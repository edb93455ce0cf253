"""On-device evaluation of a training ensemble (SURVEY §8 f3): the quantities the reference computes per exported
dictionary on the CPU — FVU (standard_metrics.py:310-314), mean L0 and per-feature activation frequency (:305-308),
features ever active (:441-454) — obtained for all M models at once from the engine's forward pass: no parameter
update and NO dense fp32 code. FVU and L0 come from the fused loss / nnz counters of the GEMM epilogues; the
per-feature activation counts are column sums of the [c > 0] activity-mask plane that the encode epilogue (or the top-k
selection) writes for the backward pass (libsce ``sce_active_counts``), accumulated over as many batches as the
held-out set has.

FVU is taken in the space the model reconstructs (the centred space for FunctionalTiedSAE with a non-trivial
centring: an orthogonal rotation leaves it unchanged, a non-uniform ``center_scale`` does not)."""
from __future__ import annotations

import contextlib
import ctypes as C
from typing import Dict, Iterable, Optional

import numpy as np
import torch

from . import _lib
from .optim import AdamConfig

EVER_ACTIVE_THRESHOLD = 10   # standard_metrics.py:446: a feature counts as "ever active" above this many rows


def evaluate(ensemble, batch: torch.Tensor, n_ever_active: bool = False, threshold: int = 0,
             counts: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """One held-out batch [B, d] (CUDA or pinned host). Returns per-model tensors on the ensemble's device:
    ``fvu``, ``mean_l0``, ``l_reconstruction``, and with ``n_ever_active`` also ``feature_counts`` ([M, n] rows on
    which each feature fired; accumulated into ``counts`` when given), ``n_ever_active`` (features that fired on
    more than ``threshold`` rows) and ``frac_dead``."""
    x = batch.to(ensemble.device, non_blocking=True).float()
    losses, aux = ensemble.forward_batch(x)
    total_var = (x - x.mean(dim=0)).pow(2).mean()
    out = {
        "l_reconstruction": losses.get("l_reconstruction", losses["loss"]),
        "mean_l0": aux["c"].count_nonzero(dim=-1).float().mean(dim=-1),
    }
    out["fvu"] = out["l_reconstruction"] / total_var
    if n_ever_active:
        counts = ensemble.active_counts(x.shape[-2], counts)
        out["feature_counts"] = counts
        out["n_ever_active"] = (counts > threshold).sum(dim=-1)
        out["frac_dead"] = 1.0 - out["n_ever_active"].float() / counts.shape[-1]
    return out


def evaluate_batches(ensemble, batches: Iterable[torch.Tensor],
                     threshold: int = EVER_ACTIVE_THRESHOLD) -> Dict[str, torch.Tensor]:
    """A held-out set streamed through in batches (``batched_calc_feature_n_ever_active``, standard_metrics.py:446-454,
    for every model of the ensemble at once, plus FVU and L0 of the whole set): FVU = sum of squared residuals / total
    variance about the set's column means — exactly the reference's formula on the concatenated set —, row-weighted
    mean L0, per-feature activation counts and frequencies, features active on more than ``threshold`` rows."""
    dev = torch.device(ensemble.device)
    sq = torch.zeros(ensemble.n_models, dtype=torch.float64, device=dev)
    l0 = torch.zeros(ensemble.n_models, dtype=torch.float64, device=dev)
    s1 = s2 = None
    rows, counts = 0, None
    for b in batches:
        x = b.to(dev, non_blocking=True).float()
        B, d = x.shape
        losses, aux = ensemble.forward_batch(x)
        sq += losses.get("l_reconstruction", losses["loss"]).double() * (B * d)
        l0 += aux["c"].count_nonzero(dim=-1).float().mean(dim=-1).double() * B
        counts = ensemble.active_counts(B, counts)
        xd = x.double()
        s1 = xd.sum(0) if s1 is None else s1 + xd.sum(0)
        s2 = xd.pow(2).sum(0) if s2 is None else s2 + xd.pow(2).sum(0)
        rows += B
    if rows == 0:
        raise ValueError("evaluate_batches needs at least one batch")
    total = (s2 - s1 * s1 / rows).sum()                      # sum over elements of (x - column mean)^2
    n_act = (counts > threshold).sum(dim=-1)
    return {"fvu": (sq / total).float(), "mean_l0": (l0 / rows).float(), "feature_counts": counts,
            "feature_frequency": counts.float() / rows, "n_ever_active": n_act,
            "frac_dead": 1.0 - n_act.float() / counts.shape[-1], "rows": rows}


# ---------------------------------------------------------------------------------------------------------------------
# Dictionary similarity (standard_metrics.py:270-303, 356-362): cosine maxima between dictionaries and the capacity of
# Scherlis et al., on the split-operand GEMM (libsce ``sce_similarity``). Each is an [n1, d] x [n2, d]^T product followed
# by a row maximum, a column maximum or a row sum; the engine keeps only those reductions, so the [n1, n2] matrix never
# exists, and one launch runs every pair of a sweep.
# ---------------------------------------------------------------------------------------------------------------------
class _Stack:
    """One side of a similarity call: fp32 [M, n, d] on a CUDA device, per-model valid rows, normalisation."""

    def __init__(self, w, rows, floor):
        self.w, self.rows, self.floor = w, rows, floor      # floor None: the matrix as given

    @property
    def models(self):
        return self.w.shape[0]


def _ld_matrix(ld):
    """(matrix [n, d], norm_floor) whose normalised rows are ``ld.get_learned_dict()``."""
    from .learned_dict import NORM_FLOOR, TiedSAE, UntiedSAE
    if isinstance(ld, TiedSAE):
        return ld.encoder, NORM_FLOOR
    if isinstance(ld, UntiedSAE):
        return ld.decoder, NORM_FLOOR
    return ld.get_learned_dict(), None       # TopKLearnedDict (stored normalised) and any other LearnedDict


def _as_stack(x):
    """FunctionalEnsemble, LearnedDict, list of LearnedDicts, or a tensor [M, n, d] / [n, d] (taken as given)."""
    from .learned_dict import LearnedDict
    if hasattr(x, "sig") and hasattr(x, "params"):                           # FunctionalEnsemble
        w, floor, rows = x.sig.learned_dict_stack(x.params, x.buffers)
        rows = None if rows is None else [int(r) for r in rows.reshape(-1).tolist()]
        return _Stack(w, rows, floor)
    if isinstance(x, LearnedDict):
        w, floor = _ld_matrix(x)
        return _Stack(w[None], None, floor)
    if isinstance(x, (list, tuple)):
        mats = [_ld_matrix(ld) if isinstance(ld, LearnedDict) else (ld, None) for ld in x]
        floors = {f for _, f in mats}
        if len(floors) != 1:                                                 # mixed kinds: normalise in torch first
            mats = [(ld.get_learned_dict() if isinstance(ld, LearnedDict) else ld, None) for ld in x]
            floors = {None}
        ns = [m.shape[0] for m, _ in mats]
        n, d = max(ns), mats[0][0].shape[1]
        if len(set(ns)) == 1:
            w = torch.stack([m for m, _ in mats])
        else:                                                                # zero-padded to the largest dictionary
            w = mats[0][0].new_zeros(len(mats), n, d)
            for i, (m, _) in enumerate(mats):
                w[i, : m.shape[0]] = m
        return _Stack(w, None if len(set(ns)) == 1 else ns, floors.pop())
    if torch.is_tensor(x):
        return _Stack(x if x.dim() == 3 else x[None], None, None)
    raise TypeError(f"expected a FunctionalEnsemble, LearnedDict(s) or a tensor, got {type(x).__name__}")


def _cuda_device(t: torch.Tensor, what: str) -> torch.device:
    """Where the engine runs ``what`` on ``t``: its device if that is a CUDA device, else the current one."""
    if t.device.type == "cuda":
        return t.device
    if not torch.cuda.is_available():
        raise RuntimeError(f"{what} runs in the sm_90a CUDA engine and needs a CUDA device; there is no CPU "
                           "implementation in the product path")
    return torch.device("cuda", torch.cuda.current_device())


def _run_similarity(a: _Stack, b: Optional[_Stack], pairs, row=True, col=True, capacity=False, arith="auto"):
    """(row_max [P, na], col_max [P, nb], capacity [Ma, na]) on the CUDA device of ``a`` (None where not requested)."""
    dev = _cuda_device(a.w, "dictionary similarity")
    code = _lib.arith_code(arith)
    prep = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()
    aw = prep(a.w)
    bw = prep(b.w) if b is not None else None
    Ma, na, d = aw.shape
    Mb, nb = (bw.shape[0], bw.shape[1]) if bw is not None else (Ma, na)
    if bw is not None and bw.shape[2] != d:
        raise ValueError(f"dictionaries of different widths: {d} and {bw.shape[2]}")
    pv = torch.as_tensor(pairs, dtype=torch.int32).reshape(-1, 2).contiguous()
    P = pv.shape[0]
    lib = _lib.load()
    need = lib.sce_similarity_workspace_bytes(Ma, na, Mb if bw is not None else 0, nb, d, P, int(capacity))
    if need == 0:
        raise ValueError(f"invalid similarity shape: a [{Ma}, {na}, {d}], b [{Mb}, {nb}], {P} pairs")
    ws, ws_ptr = _lib.workspace(need, dev, "sce_similarity_workspace_bytes")
    row_max = torch.empty(P, na, dtype=torch.float32, device=dev) if row else None
    col_max = torch.empty(P, nb, dtype=torch.float32, device=dev) if col else None
    cap = torch.full((Ma, na), float("nan"), dtype=torch.float32, device=dev) if capacity else None
    ints = lambda v: (C.c_int * len(v))(*v) if v is not None else None
    ptr = lambda t: t.data_ptr() if t is not None else None
    side = lambda s: (ints(s.rows), C.c_float(s.floor or 0.0), int(s.floor is not None))
    a_rows, a_floor, a_norm = side(a)
    b_rows, b_floor, b_norm = side(b) if b is not None else (None, C.c_float(0.0), 0)
    with torch.cuda.device(dev):
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _lib.check(lib.sce_similarity(
            aw.data_ptr(), Ma, na, a_rows, a_floor, a_norm, ptr(bw), Mb, nb, b_rows, b_floor, b_norm, d,
            pv.numpy().ctypes.data_as(C.c_void_p), P, code, ptr(row_max), ptr(col_max), ptr(cap),
            ws_ptr, need, stream), "sce_similarity")
    return row_max, col_max, cap


def _pair_list(pairs, Ma, Mb, same):
    if isinstance(pairs, str):
        if pairs == "lower":
            if not same:
                raise ValueError('pairs="lower" compares the models of one stack with each other: pass b=None')
            return [(i, j) for i in range(Ma) for j in range(i)]
        if pairs == "all":
            return [(i, j) for i in range(Ma) for j in range(Mb)]
        raise ValueError(f'pairs must be "lower", "all" or a list of (i, j), got {pairs!r}')
    return [(int(i), int(j)) for i, j in torch.as_tensor(pairs).reshape(-1, 2).tolist()]


def _valid_mean(v: torch.Tensor, rows) -> torch.Tensor:
    """Mean of each row of ``v`` [P, n] over its first ``rows[p]`` entries."""
    r = torch.as_tensor(rows, device=v.device).reshape(-1, 1)
    mask = torch.arange(v.shape[1], device=v.device)[None, :] < r
    return torch.where(mask, v, torch.zeros((), device=v.device)).sum(dim=1) / r.reshape(-1).to(v.dtype)


def dictionary_similarity(a, b=None, pairs="lower", arith: str = "auto") -> Dict[str, torch.Tensor]:
    """Cosine maxima of every chosen pair of dictionaries in one launch (the grids of big_sweep.py:108-138 and of the
    plotting scripts). ``a`` / ``b``: FunctionalEnsembles, lists of LearnedDicts (dictionaries of different sizes are
    zero-padded and masked) or tensors [M, n, d] / [n, d] taken as given (a raw truth matrix). ``b=None`` compares
    ``a`` with itself. ``pairs``: "lower" (i > j, b=None), "all" (every (i, j)) or a list of (i, j).

    Returns, on the device of ``a``:
      ``pairs``  [P, 2] (int64)
      ``mcs_ab`` [P, na]: for each atom of a[i] its best cosine in b[j] (``mcs_duplicates(b[j], a[i])``)
      ``mcs_ba`` [P, nb]: for each atom of b[j] its best cosine in a[i] (``mcs_duplicates(a[i], b[j])``)
      ``mmcs``   [Ma, Mb]: mmcs[i, j] = mean of mcs_ab over the atoms of a[i]; with b=None also mmcs[j, i] = mean of
                 mcs_ba for each pair (i, j) whose mirror is not itself a pair. Entries no pair covers are NaN.
    Entries of atoms beyond a model's dictionary size are NaN."""
    A = _as_stack(a)
    B = _as_stack(b) if b is not None else None
    Mb = B.models if B is not None else A.models
    plist = _pair_list(pairs, A.models, Mb, B is None)
    if not plist:
        raise ValueError("no pairs to compare")
    row_max, col_max, _ = _run_similarity(A, B, plist, arith=arith)
    dev = row_max.device
    pt = torch.tensor(plist, dtype=torch.long)
    na, nb = row_max.shape[1], col_max.shape[1]
    ra = A.rows or [na] * A.models
    rb = (B.rows or [nb] * B.models) if B is not None else ra
    mean_ab = _valid_mean(row_max, [ra[i] for i, _ in plist])
    mean_ba = _valid_mean(col_max, [rb[j] for _, j in plist])
    mm = torch.full((A.models, Mb), float("nan"), dtype=torch.float32, device=dev)
    ii, jj = pt[:, 0].to(dev), pt[:, 1].to(dev)
    if B is None:
        covered = set(plist)
        mirror = torch.tensor([(j, i) not in covered for i, j in plist], device=dev)
        mm[jj[mirror], ii[mirror]] = mean_ba[mirror]
    mm[ii, jj] = mean_ab
    out_dev = _input_device(a)
    return {"pairs": pt.to(out_dev), "mcs_ab": row_max.to(out_dev), "mcs_ba": col_max.to(out_dev), "mmcs": mm.to(out_dev)}


def capacity(a, arith: str = "auto") -> torch.Tensor:
    """capacity_per_feature (standard_metrics.py:356-362, Scherlis et al. 2022) of every model of ``a`` (as in
    :func:`dictionary_similarity`): [M, n], NaN beyond a model's dictionary size and for zero rows (as the reference)."""
    A = _as_stack(a)
    _, _, cap = _run_similarity(A, None, [(m, m) for m in range(A.models)], row=False, col=False, capacity=True,
                                arith=arith)
    return cap.to(_input_device(a))


def _input_device(x):
    if hasattr(x, "sig") and hasattr(x, "params"):
        return torch.device(x.device)
    if torch.is_tensor(x):
        return x.device
    if isinstance(x, (list, tuple)):
        return _input_device(x[0])
    return _ld_matrix(x)[0].device


# drop-ins with the reference's names, argument order and results (standard_metrics.py:270-303, 356-362); ``arith``
# is the engine's operand arithmetic (sce_arith)
def mcs_duplicates(ground, model, arith: str = "auto") -> torch.Tensor:
    """For each atom of ``model``, its largest cosine with an atom of ``ground``: [n_model]."""
    rm, _, _ = _run_similarity(_as_stack(model), _as_stack(ground), [(0, 0)], col=False, arith=arith)
    return rm[0].to(_input_device(model))


def mmcs(model, model2, arith: str = "auto") -> torch.Tensor:
    return mcs_duplicates(model, model2, arith=arith).mean()


def mcs_to_fixed(model, truth: torch.Tensor, arith: str = "auto") -> torch.Tensor:
    """For each atom of ``model``, its largest dot product with a row of ``truth`` as given (not normalised)."""
    rm, _, _ = _run_similarity(_as_stack(model), _Stack(truth[None], None, None), [(0, 0)], col=False, arith=arith)
    return rm[0].to(_input_device(model))


def mmcs_to_fixed(model, truth: torch.Tensor, arith: str = "auto") -> torch.Tensor:
    return mcs_to_fixed(model, truth, arith=arith).mean()


def mmcs_from_list(ld_list, arith: str = "auto") -> torch.Tensor:
    """[n, n]: 1 on the diagonal, [i, j] = [j, i] = mmcs(ld_list[i], ld_list[j]) for j < i."""
    n = len(ld_list)
    dev = _input_device(ld_list)
    out = torch.eye(n, device=dev)
    if n < 2:
        return out
    res = dictionary_similarity(list(ld_list), None, pairs="lower", arith=arith)
    sizes = [(ld if torch.is_tensor(ld) else _ld_matrix(ld)[0]).shape[0] for ld in ld_list]
    # mmcs(ld[i], ld[j]) averages, over the atoms of ld[j], their best match in ld[i]: the column maxima of (i, j)
    vals = _valid_mean(res["mcs_ba"].to(dev), [sizes[j] for _, j in res["pairs"].tolist()])
    p = res["pairs"].to(dev)
    out[p[:, 0], p[:, 1]] = vals
    out[p[:, 1], p[:, 0]] = vals
    return out


def representedness(features: torch.Tensor, model, arith: str = "auto") -> torch.Tensor:
    """For each row of ``features`` (as given), its largest dot product with an atom of ``model``: [n_features]."""
    rm, _, _ = _run_similarity(_Stack(features[None], None, None), _as_stack(model), [(0, 0)], col=False, arith=arith)
    return rm[0].to(features.device)


def capacity_per_feature(model, arith: str = "auto") -> torch.Tensor:
    return capacity(model, arith=arith)[0]


# ---------------------------------------------------------------------------------------------------------------------
# Scoring exported dictionaries on a set of activations (standard_metrics.py:305-314, 344-345, 446-454, 482-511): FVU,
# activation counts and per-feature moments of every dictionary in one pass over the activations (libsce
# ``sce_forward_stats``). Dictionaries of one kind, padded size, width and centring share one forward-only plan; the
# code [B, n] exists only as the engine's operand planes, and the moments are summed from it in the encode epilogue.
# ---------------------------------------------------------------------------------------------------------------------
_EVAL_ROWS = 8192          # rows per engine call


def _eval_kind(ld) -> str:
    from .ica import ICAEncoder
    from .learned_dict import IdentityReLU, LearnedDict, RandomDict, TiedSAE, UntiedSAE
    from .topk_encoder import TopKLearnedDict
    if isinstance(ld, TiedSAE):
        if not getattr(ld, "norm_encoder", True):
            raise NotImplementedError("TiedSAE(norm_encoder=False) is not implemented in the engine: its encoder rows "
                                      "are used unnormalised, which no engine variant computes")
        return "tied"
    if isinstance(ld, (UntiedSAE, IdentityReLU)):
        return "untied"
    if isinstance(ld, TopKLearnedDict):
        return "topk"
    if isinstance(ld, RandomDict):
        return "random"
    if isinstance(ld, ICAEncoder):
        return "ica"
    name = type(ld).__name__ if isinstance(ld, LearnedDict) else repr(type(ld))
    raise NotImplementedError(f"{name} has no engine variant: dictionary evaluation runs TiedSAE (norm_encoder=True), "
                              "UntiedSAE, TopKLearnedDict, ICAEncoder, RandomDict and IdentityReLU, and has no slow path "
                              "for other dictionaries")


def _sae_inputs(ld):
    """(encoder [n, d], bias [n], decoder [n, d] or None, translation [d] or None) of the forward-only plan that computes
    the SAE-kind dictionary ``ld``: code = flags(x - t) E^T + b), reconstruction code D. The plan's kind supplies the
    flags (``_lib.SIGNATURES``); the translation belongs to ``encode``, so the raw-batch passes apply it as well."""
    from .ica import ICAEncoder
    from .learned_dict import IdentityReLU, RandomDict, TiedSAE
    if isinstance(ld, TiedSAE):
        return ld.encoder, ld.encoder_bias, None, None
    if isinstance(ld, IdentityReLU):
        eye = torch.eye(ld.n_feats, device=ld.bias.device)
        return eye, ld.bias, eye, None
    if isinstance(ld, RandomDict):
        return ld.encoder, ld.encoder_bias, ld.encoder, None
    if isinstance(ld, ICAEncoder):
        # encode = ((x - mean) / scale - ica.mean) C^T = (x - t) (C / scale)^T with t = mean + scale * ica.mean; t is
        # subtracted from the batch, not folded into the bias: x E^T - E t would cancel on columns whose mean is far
        # larger than their spread
        f64 = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
        comp, mean, scale = f64(ld.ica.components_), f64(ld.scaler.mean_), f64(ld.scaler.scale_)
        enc = (comp / scale[None, :]).float()
        t = (mean + scale * f64(ld.ica.mean_)).float()
        return enc, torch.zeros(enc.shape[0]), ld.get_learned_dict(), t
    return ld.encoder, ld.encoder_bias, ld.decoder, None          # UntiedSAE


def _is_centred(ld) -> bool:
    if hasattr(ld, "initialize_missing"):
        ld.initialize_missing()
    t, r, s = ld.center_trans, ld.center_rot, ld.center_scale
    return not (bool((t == 0).all()) and bool((s == 1).all())
                and bool((r == torch.eye(r.shape[0], device=r.device, dtype=r.dtype)).all()))


def _eval_groups(lds, centre: bool, multiple: int):
    """Input dictionaries -> ordered {(kind, padded n, d, centred): [input index, ...]}. ``multiple``: the padded
    dictionary size is a multiple of it (8, or 16 for f16f8). Raises for what the engine does not run."""
    groups = {}
    for i, ld in enumerate(lds):
        kind = _eval_kind(ld)
        n, d = int(ld.n_feats), int(ld.activation_size)
        if d % 8:
            raise ValueError(f"dictionary {i}: activation width d = {d} must be a multiple of 8")
        topk = _lib.SIGNATURES[kind].topk
        if topk and not 0 < int(ld.sparsity) <= n:
            raise ValueError(f"dictionary {i}: sparsity must be in [1, {n}], got {ld.sparsity}")
        if topk and n % multiple:
            raise ValueError(f"dictionary {i}: a TopKLearnedDict needs n ({n}) to be a multiple of {multiple}: its rows "
                             "are normalised without a clamp, so zero padding rows would become NaN")
        if kind == "ica" and (ld.ica is None or n != ld.ica.components_.shape[0]):
            raise ValueError(f"dictionary {i}: an ICAEncoder is evaluated with n_feats equal to its fitted components' "
                             f"count, got n_feats = {n}" + ("" if ld.ica is None else
                                                             f" and {ld.ica.components_.shape[0]} components"))
        n_pad = -(-n // multiple) * multiple
        centred = centre and _lib.SIGNATURES[kind].centering and _is_centred(ld)
        groups.setdefault((kind, n_pad, d, centred), []).append(i)
    return groups


class _DictPlan:
    """The forward-only plan of one group of dictionaries (a key of :func:`_eval_groups`), prepared on ``dev``."""

    def __init__(self, key, lds, batch_max, arith, dev):
        kind, n_pad, d, centred = key
        M = len(lds)
        self.kind, self.M, self.n, self.d, self.centred, self.dev = kind, M, n_pad, d, centred, dev
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32)

        def stack(ts):
            out = torch.zeros((M, n_pad) + tuple(ts[0].shape[1:]), dtype=torch.float32, device=dev)
            for m, t in enumerate(ts):
                out[m, : t.shape[0]] = f32(t)
            return out

        sig = _lib.SIGNATURES[kind]
        params, buffers = {}, {}
        self.shift = None        # [M, d]: the translation each model's encode subtracts from the batch (ICAEncoder)
        if sig.topk:
            params["dict"] = stack([ld.dict for ld in lds])
            buffers["sparsity"] = torch.tensor([int(ld.sparsity) for ld in lds], dtype=torch.int64, device=dev)
        else:
            enc, bias, dec, shift = zip(*(_sae_inputs(ld) for ld in lds))
            params["encoder"] = stack(enc)
            params["encoder_bias"] = stack(bias)
            if sig.decoder:
                params["decoder"] = stack(dec)
            if shift[0] is not None:
                self.shift = torch.stack([f32(t) for t in shift]).contiguous()
            sizes = [int(ld.n_feats) for ld in lds]
            if any(k < n_pad for k in sizes):       # padding rows: the masked variants' coef_mask (1 = unused)
                buffers["coef_mask"] = (torch.arange(n_pad, device=dev)[None, :] >= torch.tensor(sizes, device=dev)[:, None]).to(torch.uint8)
        if centred:
            self.trans = buffers["center_trans"] = torch.stack([f32(ld.center_trans) for ld in lds]).contiguous()
            self.rot = buffers["center_rot"] = torch.stack([f32(ld.center_rot) for ld in lds]).contiguous()
            self.scale = buffers["center_scale"] = torch.stack([f32(ld.center_scale) for ld in lds]).contiguous()
        # sce_prepare and the forward-only passes never read the Adam moments; the plan only requires their pointers
        moments = dict.fromkeys(params, torch.zeros(1, dtype=torch.float32, device=dev))
        self.desc, b, keep = _lib.plan_structs(sig, params, buffers, moments, moments, batch_max=batch_max,
                                               x_per_model=centred or self.shift is not None, centering=int(centred), adam=AdamConfig(lr=0.0),
                                               adam_count_mode="frozen_t1", fwd_passes=3, bwd_passes=3, arith=arith)
        self._keep_alive = (params, buffers, moments, keep)
        self.plan, self._plan_ws = _lib.create_plan(self.desc, b, dev)
        self.stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        try:
            _lib.check(_lib.load().sce_prepare(self.plan, self.stream), "sce_prepare")
        except Exception:
            self.close()
            raise

    def batch(self, x):
        """The batch the plan reads for the rows ``x`` [B, d]: ``x`` itself, or [M, B, d] rows x - shift[m]."""
        return x if self.shift is None else (x[None] - self.shift[:, None]).contiguous()

    def bad(self) -> bool:
        flag, amax = C.c_int(0), C.c_float(0.0)
        _lib.check(_lib.load().sce_health(self.plan, C.byref(flag), C.byref(amax), self.stream), "sce_health")
        return bool(flag.value)

    def close(self):
        if getattr(self, "plan", None) is not None and self.plan.value:
            _lib.load().sce_plan_destroy(self.plan)
        self.plan = None


class _StatsPlan(_DictPlan):
    """A dictionary plan with the statistics accumulators of :func:`evaluate_dicts`."""

    def __init__(self, key, lds, batch_max, arith, dev, interference=False):
        super().__init__(key, lds, batch_max, arith, dev)
        M, n = self.M, self.n
        self.ws_bytes = _lib.load().sce_forward_stats_workspace_bytes(C.byref(self.desc), batch_max)
        self._pass_ws, self.ws_ptr = _lib.workspace(self.ws_bytes, dev, "sce_forward_stats_workspace_bytes")
        z = lambda dt: torch.zeros(M, n, dtype=dt, device=dev)
        self.sums = torch.zeros(M, n, 4, dtype=torch.float64, device=dev)
        self.seg_counts, self.seg_open, self.counts = z(torch.int32), z(torch.int32), z(torch.int32)
        self.sq = torch.zeros(M, dtype=torch.float64, device=dev)
        self.l0 = torch.zeros(M, dtype=torch.float64, device=dev)
        self.losses = torch.empty(M, _lib.SCE_LOSS_COLS, dtype=torch.float32, device=dev)
        self.nnz = torch.empty(M, dtype=torch.float32, device=dev)
        self.batch_max = batch_max
        self.cap_sums = self.nz_counts = None
        if interference:     # the expected interference of each call's code (sce_code_interference)
            self.if_bytes = _lib.load().sce_interference_workspace_bytes(C.byref(self.desc), batch_max)
            self._if_ws, self.if_ptr = _lib.workspace(self.if_bytes, dev, "sce_interference_workspace_bytes")
            self.cap_sums = torch.zeros(M, n, dtype=torch.float64, device=dev)
            self.nz_counts = torch.zeros(M, n, dtype=torch.int64, device=dev)

    def run(self, x, seg, phase):
        lib = _lib.load()
        B, d = x.shape
        x_hat = torch.empty(self.M, B, d, dtype=torch.float32, device=self.dev) if self.centred else None
        _lib.check(lib.sce_forward_stats(
            self.plan, self.batch(x).data_ptr(), B, seg, phase, x_hat.data_ptr() if x_hat is not None else None,
            self.losses.data_ptr(), self.nnz.data_ptr(), self.sums.data_ptr(), self.seg_counts.data_ptr(),
            self.seg_open.data_ptr(), self.ws_ptr, self.ws_bytes, self.stream), "sce_forward_stats")
        _lib.check(lib.sce_active_counts(self.plan, B, self.counts.data_ptr(), self.stream), "sce_active_counts")
        if self.cap_sums is not None:
            _lib.check(lib.sce_code_interference(self.plan, B, self.cap_sums.data_ptr(), self.nz_counts.data_ptr(),
                                                 self.if_ptr, self.if_bytes, self.stream), "sce_code_interference")
        if x_hat is None:
            self.sq += self.losses[:, 1].double() * (B * d)
        else:       # the reference's residual x - uncenter(x^_c), in the raw space (standard_metrics.py:310-314)
            r = (x[None] - self.trans[:, None]) - torch.bmm(x_hat / self.scale[:, None], self.rot)
            self.sq += r.double().pow(2).sum(dim=(1, 2))
        self.l0 += self.nnz.double() * B

    def start_split(self, top):
        """Ready the pass of the top- and rest-feature errors: ``top`` [M, n_top] int64, the chosen features per model.
        The statistics pass is over, so its workspace gives way to this one."""
        M, n_top = top.shape
        self.n_top, self.top = n_top, top
        self.top_cols = top.to(torch.int32).contiguous()
        self._pass_ws = None
        self.split_bytes = _lib.load().sce_forward_split_workspace_bytes(C.byref(self.desc), self.batch_max, n_top)
        self._split_ws, self.split_ptr = _lib.workspace(self.split_bytes, self.dev, "sce_forward_split_workspace_bytes")
        self.sq_top = torch.zeros(M, dtype=torch.float64, device=self.dev)
        self.sq_rest = torch.zeros(M, dtype=torch.float64, device=self.dev)

    def run_split(self, x):
        B, d = x.shape
        x_hat = x_hat_top = None
        if self.centred:
            x_hat = torch.empty(self.M, B, d, dtype=torch.float32, device=self.dev)
            x_hat_top = torch.empty_like(x_hat)
        ptr = lambda t: t.data_ptr() if t is not None else None
        _lib.check(_lib.load().sce_forward_split(
            self.plan, self.batch(x).data_ptr(), B, self.n_top, self.top_cols.data_ptr(), self.sq_top.data_ptr(),
            self.sq_rest.data_ptr(), ptr(x_hat), ptr(x_hat_top), self.split_ptr, self.split_bytes, self.stream),
            "sce_forward_split")
        if self.centred:
            # the reference applies center (not uncenter) to both partial reconstructions, then compares them with the
            # raw batch (standard_metrics.py:335-339; SURVEY Q14)
            cen = lambda v: torch.bmm(v - self.trans[:, None], self.rot.transpose(1, 2)) * self.scale[:, None]
            self.sq_top += (x[None] - cen(x_hat_top)).double().pow(2).sum(dim=(1, 2))
            self.sq_rest += (x[None] - cen(x_hat - x_hat_top)).double().pow(2).sum(dim=(1, 2))


def _top_features(sums, n):
    """The ``n_top`` features of largest mean code among the first ``n``, from the fp64 code sums [n_pad]: descending,
    equal sums ordered by the lower feature index."""
    return torch.sort(sums[:n], descending=True, stable=True).indices


def _check_n_top(n_top, lds):
    if n_top is None:
        return None
    if isinstance(n_top, bool) or not isinstance(n_top, (int, np.integer)):
        raise ValueError(f"n_top must be an integer, got {n_top!r}")
    n_top = int(n_top)
    if not 1 <= n_top <= _lib.SCE_SPLIT_MAX_TOP:
        raise ValueError(f"n_top must lie in [1, {_lib.SCE_SPLIT_MAX_TOP}], got {n_top}")
    for i, ld in enumerate(lds):
        if n_top > int(ld.n_feats):
            raise ValueError(f"n_top = {n_top} exceeds dictionary {i}'s {int(ld.n_feats)} features")
    return n_top


def _dict_inputs(learned_dicts, activations, arith, centre):
    """(LearnedDicts, groups of :func:`_eval_groups`, arithmetic that runs) of a forward-only pass of
    ``learned_dicts`` (LearnedDicts or ``(LearnedDict, hparams)`` pairs) over ``activations``; raises for what the
    engine does not run."""
    _lib.arith_code(arith)
    lds = [ld[0] if isinstance(ld, (tuple, list)) else ld for ld in learned_dicts]
    if not lds:
        raise ValueError("no dictionaries to evaluate")
    if activations.dim() != 2 or activations.shape[0] == 0:
        raise ValueError(f"activations must be a non-empty [N, d] tensor, got shape {tuple(activations.shape)}")
    if activations.dtype not in (torch.float32, torch.float16):
        raise ValueError(f"activations must be fp32 or fp16, got {activations.dtype}")
    # AUTO runs bf16x3: the fp32 range, so activations fp16 cannot hold give finite results
    ar = "bf16x3" if arith == "auto" else arith
    groups = _eval_groups(lds, centre, 16 if ar == "f16f8" else 8)
    for (kind, n_pad, dd, _), idx in groups.items():
        if dd != activations.shape[1]:
            raise ValueError(f"dictionary {idx[0]} has width {dd}, the activations {activations.shape[1]}")
    return lds, groups, ar


@contextlib.contextmanager
def _plans(groups, lds, dev, make):
    """[(plan, input indices)]: ``make(key, dictionaries)`` of every group, under ``dev``. Every plan built is closed on
    exit, also when building a later one fails."""
    plans = []
    with torch.cuda.device(dev):
        try:
            for key, idx in groups.items():
                plans.append((make(key, [lds[i] for i in idx]), idx))
            yield plans
        finally:
            for p, _ in plans:
                p.close()


def _check_f16f8_range(plans, arith):
    """After a pass: raise if f16f8 met a value outside its fp16 plane's range."""
    if arith == "f16f8" and any(p.bad() for p, _ in plans):
        raw = [p for p, _ in plans if p.bad() and _lib.SIGNATURES[p.kind].decoder_raw]
        where = "the activations or a RandomDict's raw decoder rows hold" if raw else "the activations hold"
        raise ValueError(f"{where} a value the f16f8 arithmetic's fp16 plane cannot (|v| >= 65520 or NaN): use "
                         "arith='bf16x3' or 'auto'")


def _to_device(out, device):
    """A result dict with its tensors on ``device``."""
    return {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in out.items()}


def _eval_rows(activations, dev, cuts):
    """The row ranges ``cuts`` of ``activations`` as fp32 [B, d] batches on ``dev``: device input sliced in place, host
    input streamed through HostBatchPrefetcher; fp16 is converted per batch on the device."""
    if activations.device.type == "cuda":
        for s, e in cuts:
            yield activations[s:e].float().contiguous()
        return
    from .train_loop import HostBatchPrefetcher
    for xb in HostBatchPrefetcher((activations[s:e] for s, e in cuts), dev):
        yield xb.float().contiguous()


def _evaluate(learned_dicts, activations, segment, threshold, arith, centre, n_top=None, interference=False):
    if int(segment) < 1:
        raise ValueError(f"batch_size / segment must be >= 1, got {segment}")
    segment = int(segment)
    if not isinstance(interference, (bool, np.bool_)):
        raise ValueError(f"interference must be True or False, got {interference!r}")
    lds, groups, ar = _dict_inputs(learned_dicts, activations, arith, centre)
    n_top = _check_n_top(n_top, lds)
    dev = _cuda_device(activations, "dictionary evaluation")
    N, d = activations.shape
    # engine calls: a multiple of the segment where one fits, and a cut where the last segment starts (its sums are
    # weighted by segment / rows, as the reference's running average does)
    rows = _EVAL_ROWS // segment * segment if segment <= _EVAL_ROWS else _EVAL_ROWS
    n_seg = -(-N // segment)
    last = (n_seg - 1) * segment
    cuts = [(s, min(s + rows, last)) for s in range(0, last, rows)] + [(s, min(s + rows, N)) for s in range(last, N, rows)]
    batch_max = max(e - s for s, e in cuts)
    results = [None] * len(lds)
    make = lambda key, g: _StatsPlan(key, g, batch_max, ar, dev, interference=bool(interference))
    with _plans(groups, lds, dev, make) as plans:
        s1 = torch.zeros(d, dtype=torch.float64, device=dev)
        s2 = torch.zeros(d, dtype=torch.float64, device=dev)
        snap = [torch.zeros_like(p.sums) for p, _ in plans]
        for (s, e), x in zip(cuts, _eval_rows(activations, dev, cuts)):
            if s == last and last > 0:
                snap = [p.sums.clone() for p, _ in plans]
            for p, _ in plans:
                p.run(x, segment, s % segment)
            xd = x.double()
            s1 += xd.sum(0)
            s2 += xd.pow(2).sum(0)
        _check_f16f8_range(plans, ar)
        if n_top is not None:
            # the second pass: each dictionary's top features from the first pass's code sums, then the two errors
            for p, idx in plans:
                top = torch.stack([_top_features(p.sums[k, :, 0], int(lds[i].n_feats))[:n_top] for k, i in enumerate(idx)])
                if p.kind == "ica":     # (no second pass: the reference's decode of its code raises, as for ``fvu``)
                    p.top = top
                else:
                    p.start_split(top)
            split = [p for p, _ in plans if p.kind != "ica"]
            if split:
                for x in _eval_rows(activations, dev, cuts):
                    for p in split:
                        p.run_split(x)
        total = (s2 - s1 * s1 / N).sum()
        r_last = N - last
        for (p, idx), sn in zip(plans, snap):
            full, tail = sn, p.sums - sn
            m = (full + (segment / r_last) * tail) / (n_seg * segment)        # [M, n, 4] fp64
            # ICAEncoder: the reference's decode of its fp64 code by the fp32 dictionary raises, so no FVU is defined
            fvu = (p.sq / total).float() if p.kind != "ica" else torch.full_like(p.sq, float("nan"), dtype=torch.float32)
            l0 = (p.l0 / N).float()
            for k, i in enumerate(idx):
                n = int(lds[i].n_feats)
                counts = p.counts[k, :n].clone()
                n_act = (counts > threshold).sum()
                mean, m2, m3, m4 = (m[k, :n, q] for q in range(4))
                var = m2 - mean * mean
                out = {"fvu": fvu[k], "mean_l0": l0[k], "feature_counts": counts,
                       "feature_frequency": counts.float() / N, "n_ever_active": n_act,
                       "frac_dead": 1.0 - n_act.float() / n, "rows": N,
                       # (the last segment is still open after the pass: its flags count as well)
                       "times_active": (p.seg_counts[k, :n] + p.seg_open[k, :n]).float(), "mean": mean.float(), "m2": m2.float(),
                       "m3": m3.float(), "m4": m4.float(), "var": var.float(),
                       "skew": (m3 / var.pow(1.5).clamp(min=1e-8)).float(),
                       "kurtosis": (m4 / var.pow(2).clamp(min=1e-8)).float()}
                if n_top is not None:
                    nan = torch.full((), float("nan"), device=dev)
                    out["top_features"] = p.top[k].clone()
                    out["fvu_top"] = (p.sq_top[k] / total).float() if p.kind != "ica" else nan
                    out["fvu_rest"] = (p.sq_rest[k] / total).float() if p.kind != "ica" else nan.clone()
                if interference:
                    out["expected_interference"] = (p.cap_sums[k, :n] / p.nz_counts[k, :n].clamp(min=1)).float()
                results[i] = _to_device(out, activations.device)
    return results


def evaluate_dicts(learned_dicts, activations: torch.Tensor, segment: int = 1000,
                   threshold: int = EVER_ACTIVE_THRESHOLD, arith: str = "auto", n_top: Optional[int] = None,
                   interference: bool = False):
    """Scores of exported dictionaries on a set of activations, in one pass for all of them.

    ``learned_dicts``: LearnedDicts or ``(LearnedDict, hparams)`` pairs (what ``torch.load("learned_dicts.pt")``
    returns): TiedSAE (norm_encoder=True, any centring), UntiedSAE, TopKLearnedDict, and the baselines ICAEncoder (its
    signed code, translation included), RandomDict (raw decoder rows) and IdentityReLU. ICAEncoder's ``fvu`` is NaN:
    the reference's decode of its fp64 code raises (SURVEY Q12). ``activations``: [N, d] fp32 or
    fp16, on the CPU (streamed to the GPU) or a CUDA device. Each dictionary encodes the centred batch, as ``predict``
    and ``mean_nonzero_activations`` do. ``arith``: the engine's operand arithmetic; "auto" runs bf16x3, which holds
    the fp32 range.

    Returns one dict per input dictionary, in input order, with tensors on the device of ``activations``:
      ``fvu``, ``mean_l0``, ``feature_counts``, ``feature_frequency``, ``n_ever_active`` (count > ``threshold``),
      ``frac_dead``, ``rows`` as :func:`evaluate_batches` (FVU with the residual in the raw space, as the reference's
      ``fraction_variance_unexplained``), and ``times_active``, ``mean``, ``m2``, ``m3``, ``m4``, ``var``, ``skew``,
      ``kurtosis`` as ``calc_moments_streaming`` with ``batch_size = segment`` defines them (standard_metrics.py:482-511:
      ``times_active`` counts segments, the last partial segment is weighted like a full one).

    With an integer ``n_top`` (1 .. 64, at most every dictionary's ``n_feats``; the reference has no such bound), a
    second pass over the activations adds the scores of ``fraction_variance_unexplained_top_activating``
    (standard_metrics.py:316-342):
      ``top_features`` [n_top] int64: the features of largest mean code over all N rows, descending, equal means
                       ordered by the lower feature index (the reference's argsort leaves their order open)
      ``fvu_top``      mean((x - x^_top)^2) / the total variance of ``fvu``, with x^_top the decode of the code on
                       ``top_features`` alone, and ``fvu_rest`` the same for the code on every other feature. As the
                       reference, a centred TiedSAE passes both decodes through ``center`` (not ``uncenter``) before
                       comparing them with the raw batch (SURVEY Q14). NaN for ICAEncoder, as ``fvu``.
    The other entries are bitwise those of a call without ``n_top``.

    With ``interference=True`` the statistics pass also adds ``expected_interference`` [n] fp32: the reference's
    ``calc_expected_interference(ld.get_learned_dict(), code)`` (big_sweep.py:43-57) over all N rows of the code the
    engine computes, on every kind (ICAEncoder's signed code included). Only each row's active features are compared,
    so the [n, n] cosine matrix is never formed (libsce ``sce_code_interference``; SURVEY Q15). The other entries are
    bitwise those of a call without it."""
    return _evaluate(learned_dicts, activations, segment, threshold, arith, centre=True, n_top=n_top,
                     interference=interference)


# drop-ins with the reference's names, argument order and results (standard_metrics.py:305-314, 344-345, 446-454,
# 482-511), on the device of the activations
def fraction_variance_unexplained(model, batch: torch.Tensor, arith: str = "auto") -> torch.Tensor:
    return _evaluate([model], batch, 1000, EVER_ACTIVE_THRESHOLD, arith, centre=True)[0]["fvu"]


def fraction_variance_unexplained_top_activating(model, batch: torch.Tensor, n_top: int = 2, arith: str = "auto"):
    """(FVU of the decode of the ``n_top`` features of largest mean code, FVU of the decode of the others), 0-dim
    tensors; see :func:`evaluate_dicts`."""
    r = _evaluate([model], batch, 1000, EVER_ACTIVE_THRESHOLD, arith, centre=True, n_top=n_top)[0]
    return r["fvu_top"], r["fvu_rest"]


_INTERFERENCE_ROWS = 8192   # code rows per sce_expected_interference call (its workspace grows with them)


def calc_expected_interference(dictionary: torch.Tensor, batch: torch.Tensor, arith: str = "auto") -> torch.Tensor:
    """big_sweep.py:43-57 on the GPU: ``dictionary`` [n, d] (its rows are normalised here with the 1e-8 clamp) and
    ``batch`` the CODE [B, n] (not the activations), both on one CUDA device. Returns [n] fp32 on that device: for
    each feature, the sum over the rows where its code is non-zero of c / max(sum_j cos^2 c_j, 1e-8), over that row
    count (at least 1). The code is used as given in fp32, so ``arith`` (checked, for the drop-ins' common signature)
    changes nothing: the cosines are fp32 FMA dot products either way."""
    _lib.arith_code(arith)
    if not torch.is_tensor(dictionary) or not torch.is_tensor(batch):
        raise TypeError("dictionary and batch must be tensors")
    if dictionary.dim() != 2 or batch.dim() != 2:
        raise ValueError(f"dictionary must be [n, d] and batch [B, n], got {tuple(dictionary.shape)} and "
                         f"{tuple(batch.shape)}")
    n, d = dictionary.shape
    if batch.shape[1] != n:
        raise ValueError(f"batch has {batch.shape[1]} features, the dictionary {n}")
    if n == 0 or d == 0 or batch.shape[0] == 0:
        raise ValueError(f"empty dictionary [{n}, {d}] or batch [{batch.shape[0]}, {n}]")
    if batch.device.type != "cuda" or dictionary.device != batch.device:
        raise ValueError("calc_expected_interference runs in the sm_90a CUDA engine: dictionary and batch must be on "
                         f"one CUDA device, got {dictionary.device} and {batch.device}")
    if not (dictionary.is_floating_point() and batch.is_floating_point()):
        raise ValueError(f"dictionary and batch must be floating point, got {dictionary.dtype} and {batch.dtype}")
    dev = batch.device
    lib = _lib.load()
    w = dictionary.detach().float().contiguous()
    rows = min(batch.shape[0], _INTERFERENCE_ROWS)
    need = lib.sce_expected_interference_workspace_bytes(n, d, rows)
    cap = torch.zeros(n, dtype=torch.float64, device=dev)
    nz = torch.zeros(n, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        ws, ws_ptr = _lib.workspace(need, dev, "sce_expected_interference_workspace_bytes")
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        for s in range(0, batch.shape[0], rows):
            c = batch[s:s + rows].detach().float().contiguous()
            _lib.check(lib.sce_expected_interference(w.data_ptr(), n, d, c.data_ptr(), c.shape[0], cap.data_ptr(),
                                                     nz.data_ptr(), ws_ptr, need, stream), "sce_expected_interference")
    return (cap / nz.clamp(min=1)).float()


def r_squared(model, batch: torch.Tensor, arith: str = "auto") -> torch.Tensor:
    return 1.0 - fraction_variance_unexplained(model, batch, arith=arith)


def mean_nonzero_activations(model, batch: torch.Tensor, arith: str = "auto") -> torch.Tensor:
    return _evaluate([model], batch, 1000, EVER_ACTIVE_THRESHOLD, arith, centre=True)[0]["feature_frequency"]


def batched_calc_feature_n_ever_active(learned_dict, activations: torch.Tensor, batch_size: int = 1000,
                                       threshold: int = 10, arith: str = "auto") -> int:
    """Features non-zero on more than ``threshold`` rows; encodes the raw activations (no ``center``)."""
    return int(_evaluate([learned_dict], activations, batch_size, threshold, arith, centre=False)[0]["n_ever_active"])


def calc_moments_streaming(learned_dict, activations: torch.Tensor, batch_size: int = 1000, arith: str = "auto"):
    """(times_active, mean, var, skew, kurtosis, m4), each [n] fp32; encodes the raw activations (no ``center``)."""
    r = _evaluate([learned_dict], activations, batch_size, EVER_ACTIVE_THRESHOLD, arith, centre=False)[0]
    return r["times_active"], r["mean"], r["var"], r["skew"], r["kurtosis"], r["m4"]


# ---------------------------------------------------------------------------------------------------------------------
# Record selection for reading what features mean (interpret.py:82-212 make_feature_activation_dataset, :265-321
# interpret): per feature, the fragments with the largest maximum and a random sample of the fragments in which it fires,
# with their per-token code values (libsce ``sce_forward_fragments``). The [N, n] code and the reference's F·L·N fp16
# tables are never formed: per engine call the fragment maxima are reduced from the operand planes, and per-feature
# lists of at most 64 entries are merged on the device.
# ---------------------------------------------------------------------------------------------------------------------
FRAGMENT_MAX_LIST = 64     # largest n_top / n_random
FRAGMENT_MAX_LEN = 8192    # largest fragment: one engine call


def _list_order(key, frag):
    """Per row, the permutation that sorts (key, frag) by key descending, then fragment ascending; empty entries
    (fragment -1) go last: float keys, which may be negative (ICAEncoder's maxima), rank them at -inf, integer keys
    (priorities, >= 0) at -1."""
    empty = frag < 0
    f = torch.where(empty, torch.iinfo(torch.int64).max, frag)
    k = torch.where(empty, torch.full_like(key, float("-inf") if key.is_floating_point() else -1), key)
    o1 = torch.sort(f, dim=-1, stable=True).indices
    o2 = torch.sort(k.gather(-1, o1), dim=-1, descending=True, stable=True).indices
    return o1.gather(-1, o2)


class _FragmentPlan(_DictPlan):
    """A dictionary plan with its fragment lists, which accumulate over engine calls."""

    def __init__(self, key, lds, batch_max, L, n_top, n_random, seed, want_act, arith, dev):
        super().__init__(key, lds, batch_max, arith, dev)
        M, n = self.M, self.n
        self.L, self.n_top, self.n_random, self.seed = L, n_top, n_random, seed
        self.ws_bytes = _lib.load().sce_fragments_workspace_bytes(C.byref(self.desc), batch_max, L)
        self._pass_ws, self.ws_ptr = _lib.workspace(self.ws_bytes, dev, "sce_fragments_workspace_bytes")
        self.top_val = torch.zeros(M, n, n_top, dtype=torch.float32, device=dev)
        self.top_frag = torch.full((M, n, n_top), -1, dtype=torch.int64, device=dev)     # -1: empty entry
        self.rnd_key = torch.zeros(M, n, n_random, dtype=torch.int64, device=dev)
        self.rnd_frag = torch.full((M, n, n_random), -1, dtype=torch.int64, device=dev)
        act = lambda k: torch.zeros(M, n, k, L, dtype=torch.float32, device=dev) if want_act and k else None
        self.top_act, self.rnd_act = act(n_top), act(n_random)
        self.n_active = torch.zeros(M, n, dtype=torch.int32, device=dev)

    def run(self, x, frag0):
        ptr = lambda t: t.data_ptr() if t is not None and t.numel() else None
        _lib.check(_lib.load().sce_forward_fragments(
            self.plan, self.batch(x).data_ptr(), x.shape[0], self.L, frag0, self.n_top, self.n_random,
            self.seed & 0xFFFFFFFFFFFFFFFF, ptr(self.top_val), ptr(self.top_frag), ptr(self.top_act), ptr(self.rnd_key),
            ptr(self.rnd_frag), ptr(self.rnd_act), self.n_active.data_ptr(), self.ws_ptr, self.ws_bytes, self.stream),
            "sce_forward_fragments")

    def results(self, k, n):
        """Model k's lists, sorted, for its first n features."""
        top_o = _list_order(self.top_val[k, :n], self.top_frag[k, :n])
        rnd_o = _list_order(self.rnd_key[k, :n], self.rnd_frag[k, :n])
        rows = lambda a, o: None if a is None else a[k, :n].gather(1, o[..., None].expand(-1, -1, self.L))
        count = self.n_active[k, :n].long()
        return {"top_values": self.top_val[k, :n].gather(1, top_o), "top_fragments": self.top_frag[k, :n].gather(1, top_o),
                "top_activations": rows(self.top_act, top_o),
                "random_fragments": self.rnd_frag[k, :n].gather(1, rnd_o), "random_activations": rows(self.rnd_act, rnd_o),
                "n_active_fragments": count, "skipped": count < self.n_random}


def top_activating_fragments(learned_dicts, activations: torch.Tensor, fragment_len: int = 64, n_top: int = 20,
                             n_random: int = 20, seed: int = 0, return_activations: bool = True, arith: str = "auto"):
    """Each feature's top-activating and random activating fragments, with their per-token code values: the records
    ``interpret()`` (interpret.py:265-321) hands to the explainer, for every dictionary in one pass.

    ``learned_dicts``: LearnedDicts or ``(LearnedDict, hparams)`` pairs (TiedSAE with norm_encoder=True, UntiedSAE,
    TopKLearnedDict, ICAEncoder, RandomDict, IdentityReLU), grouped, padded and streamed as :func:`evaluate_dicts` does. ``activations``: [N, d] fp32 or
    fp16, on the CPU (streamed to the GPU) or a CUDA device, in sequence order: fragment g is rows
    g·L … g·L+L−1, L = ``fragment_len`` (a multiple of 32 in [32, 8192]; N must be a multiple of it). The raw rows are
    encoded, with no ``center()``, as make_feature_activation_dataset does. ``arith``: "auto" runs bf16x3; "f16f8"
    raises on values fp16 cannot hold.

    Per feature f, with c the code and the fragment maximum max_t c[g·L+t, f] (>= 0; ICAEncoder's signed code may give
    negative maxima, and "active" below means c != 0 on some row, where the reference tests the maximum for 0):
      top records     the ``n_top`` fragments with the largest maximum, descending, ties broken by the lower fragment
                      index; zero-maximum fragments fill the list when fewer are positive, as the reference's
                      ``sort_values(...).head(20)``. The engine's fp32 values are ranked, where the reference sorts its
                      fp16 table with a quicksort that leaves the order of ties unspecified.
      random records  up to ``n_random`` ACTIVE fragments (c > 0 on some row, from the engine's activity mask), drawn
                      uniformly without replacement, in draw order: the fragments sorted by a priority
                      splitmix64(splitmix64(splitmix64(seed) ^ f) ^ g) >> 1, descending, ties broken by fragment.
                      This is the distribution of the reference's fresh permutation per feature popped until 20 active
                      fragments are found, not its draws. The reference tests its fp16 maximum for 0 instead of the
                      activity, which differs only for maxima below fp16's smallest subnormal (2^-24).
      skipped         fewer than ``n_random`` active fragments (the reference's ``skip_feature``).
    The per-token values are the code as the engine holds it (the joined operand planes for the SAE kinds, relu(score)
    under the activity mask for top-k), and ``top_values[f, i] == top_activations[f, i].max()`` bitwise.

    Returns one dict per input dictionary, in input order, on the device of ``activations``: ``top_values`` [n, n_top]
    fp32, ``top_fragments`` [n, n_top] int64, ``top_activations`` [n, n_top, L] fp32, ``random_fragments``
    [n, n_random] int64 (-1 where unfilled, with zero activations), ``random_activations`` [n, n_random, L] fp32,
    ``n_active_fragments`` [n] int64, ``skipped`` [n] bool and ``fragments`` = N / L. With fewer than ``n_top``
    fragments in all, the top list ends in entries with fragment -1 and value 0. ``return_activations=False`` leaves
    the two activation entries None and skips their copies.

    Memory: the per-token records take n·(n_top + n_random)·L·4 bytes per dictionary on the device — 671 MB for
    config 2's 16 dictionaries of 4096 features at 20 + 20 and L = 64."""
    L, n_top, n_random = int(fragment_len), int(n_top), int(n_random)
    if L < 32 or L > FRAGMENT_MAX_LEN or L % 32:
        raise ValueError(f"fragment_len must be a multiple of 32 in [32, {FRAGMENT_MAX_LEN}], got {fragment_len}")
    for name, v in (("n_top", n_top), ("n_random", n_random)):
        if v < 0 or v > FRAGMENT_MAX_LIST:
            raise ValueError(f"{name} must lie in [0, {FRAGMENT_MAX_LIST}], got {v}")
    if n_top + n_random == 0:
        raise ValueError("n_top and n_random are both 0: there is nothing to select")
    lds, groups, ar = _dict_inputs(learned_dicts, activations, arith, False)
    N = activations.shape[0]
    if N % L:
        raise ValueError(f"the activations' {N} rows are not a whole number of fragments of {L} rows")
    dev = _cuda_device(activations, "fragment selection")
    rows = min(_EVAL_ROWS // L * L, N)          # engine calls are cut at fragment boundaries
    cuts = [(s, min(s + rows, N)) for s in range(0, N, rows)]
    results = [None] * len(lds)
    make = lambda key, g: _FragmentPlan(key, g, rows, L, n_top, n_random, int(seed), return_activations, ar, dev)
    with _plans(groups, lds, dev, make) as plans:
        for (s, e), x in zip(cuts, _eval_rows(activations, dev, cuts)):
            for p, _ in plans:
                p.run(x, s // L)
        _check_f16f8_range(plans, ar)
        for p, idx in plans:
            for k, i in enumerate(idx):
                out = p.results(k, int(lds[i].n_feats))
                out["fragments"] = N // L
                results[i] = _to_device(out, activations.device)
    return results
