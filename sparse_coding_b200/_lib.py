"""ctypes binding of libsce.so (include/sce.h). No torch types cross this boundary: only integers, floats and raw
device pointers (``tensor.data_ptr()``).

The library is built in-tree (``make`` / ``__graft_entry__.build()``) next to this file. There is NO fallback:
if it is missing, or the process has no sm_90 device when a plan is created, the engine raises."""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import torch

from .optim import AdamConfig

_HERE = os.path.dirname(os.path.abspath(__file__))
# SCE_LIB: an alternative build of the same library (kernel A/B experiments)
LIB_PATH = os.environ.get("SCE_LIB") or os.path.join(_HERE, "libsce.so")

SCE_TIED, SCE_UNTIED, SCE_TOPK, SCE_TIED_LEARNED_CENTER = 0, 1, 2, 3
SCE_CODE_LINEAR, SCE_DECODER_RAW = 1 << 8, 1 << 9     # forward-only modifiers of SCE_UNTIED, or'ed into desc.variant
SCE_SPLIT_MAX_TOP = 64      # largest n_top of sce_forward_split
SCE_ADAM_FROZEN_T1, SCE_ADAM_STANDARD = 0, 1
SCE_LOSS_COLS = 4
SCE_ARITH_AUTO, SCE_ARITH_BF16X3, SCE_ARITH_F16F8 = 0, 1, 2
ARITH_CODE = {"auto": SCE_ARITH_AUTO, "bf16x3": SCE_ARITH_BF16X3, "f16f8": SCE_ARITH_F16F8}
ARITH_NAME = {SCE_ARITH_BF16X3: "bf16x3", SCE_ARITH_F16F8: "f16f8"}

# every symbol include/sce.h declares (tests check that the built library exports all of them)
EXPORTS = [
    "sce_version", "sce_last_error", "sce_workspace_bytes", "sce_plan_create", "sce_plan_destroy", "sce_prepare",
    "sce_step", "sce_step_host", "sce_forward", "sce_read_code", "sce_grads", "sce_gather_rows",
    "sce_last_launch_count", "sce_get_step_count", "sce_set_step_count", "sce_profile_begin", "sce_profile_end",
    "sce_plan_arith", "sce_input_absmax", "sce_health", "sce_clear_health", "sce_active_counts",
    "sce_similarity_workspace_bytes", "sce_similarity", "sce_forward_stats_workspace_bytes", "sce_forward_stats",
    "sce_fragments_workspace_bytes", "sce_forward_fragments", "sce_forward_split_workspace_bytes", "sce_forward_split",
    "sce_interference_workspace_bytes", "sce_code_interference", "sce_expected_interference_workspace_bytes",
    "sce_expected_interference", "sce_cross_moments_workspace_bytes", "sce_cross_moments", "sce_correlation_finish",
    "sce_synth_rows", "sce_read_center_grad",
    "sce_second_moments_workspace_bytes", "sce_second_moments", "sce_ica_pass_workspace_bytes", "sce_ica_pass",
    "sce_nmf_project_workspace_bytes", "sce_nmf_project", "sce_nmf_grams_workspace_bytes", "sce_nmf_grams",
    "sce_nmf_cd_sweep_workspace_bytes", "sce_nmf_cd_sweep", "sce_nmf_residual_workspace_bytes", "sce_nmf_residual",
    "sce_track_workspace_bytes", "sce_step_tracked", "sce_resample",
]
PHASES = ["split", "encode", "decode", "losses", "dcode", "dw", "adam"]


class SceDesc(C.Structure):
    _fields_ = [
        ("variant", C.c_int), ("n_models", C.c_int), ("d", C.c_int), ("n", C.c_int), ("batch_max", C.c_int),
        ("x_per_model", C.c_int),
        ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float), ("eps_root", C.c_float),
        ("adam_count_mode", C.c_int), ("fwd_passes", C.c_int), ("bwd_passes", C.c_int), ("norm_floor", C.c_float),
        ("arith", C.c_int), ("topk_k_max", C.c_int), ("centering", C.c_int),
        ("encoder_nonneg", C.c_int), ("input_shift", C.c_float),
    ]


class SceBuffers(C.Structure):
    _fields_ = [
        ("encoder", C.c_void_p), ("encoder_bias", C.c_void_p), ("decoder", C.c_void_p),
        ("encoder_m", C.c_void_p), ("encoder_v", C.c_void_p), ("bias_m", C.c_void_p), ("bias_v", C.c_void_p),
        ("decoder_m", C.c_void_p), ("decoder_v", C.c_void_p),
        ("l1_alpha", C.c_void_p), ("bias_decay", C.c_void_p), ("coef_mask", C.c_void_p), ("sparsity", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
        ("center_trans", C.c_void_p), ("center_rot", C.c_void_p), ("center_scale", C.c_void_p),
        ("center", C.c_void_p), ("center_m", C.c_void_p), ("center_v", C.c_void_p),
    ]


class SceTrack(C.Structure):
    _fields_ = [
        ("err", C.c_void_p), ("serial", C.c_void_p), ("rows", C.c_void_p), ("filled", C.c_void_p),
        ("counts", C.c_void_p), ("next_serial", C.c_longlong), ("n_worst", C.c_int),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
    ]


@dataclass(frozen=True)
class EngineSignature:
    """What one engine-backed signature (``DictSignature.variant``) puts into ``SceDesc`` / ``SceBuffers``."""
    variant: int                 # sce_variant
    main: str                    # the parameter the engine trains as its (first) dictionary
    loss_keys: tuple             # the loss columns it reports (of "loss", "l_reconstruction", "l_l1", "l_bias_decay")
    decoder: bool = False        # a separate decoder (untied)
    bias_decay: bool = False     # the engine adds buffers["bias_decay"] to the loss
    learned_center: bool = False   # params["center"], trained with its Adam moments
    centering: bool = False      # FunctionalTiedSAE's centring buffers (center_trans / center_rot / center_scale)
    encoder_nonneg: bool = False   # the dictionary is max(E, 0)
    input_shift: float = 0.0     # encode and reconstruct x + input_shift
    norm_floor: float = 1e-8     # clamp of the dictionary's row norms (0: none)
    topk: bool = False           # buffers["sparsity"] holds each model's k; no bias, no sparsity penalty
    code_linear: bool = False    # forward-only: the code is x E^T + b, no clamp (SCE_CODE_LINEAR)
    decoder_raw: bool = False    # forward-only: the decoder's rows as given, not normalised (SCE_DECODER_RAW)


_SAE_LOSSES = ("loss", "l_reconstruction", "l_l1")
SIGNATURES = {
    "tied": EngineSignature(SCE_TIED, "encoder", _SAE_LOSSES, bias_decay=True, centering=True),
    "masked_tied": EngineSignature(SCE_TIED, "encoder", _SAE_LOSSES),
    "untied": EngineSignature(SCE_UNTIED, "encoder", _SAE_LOSSES + ("l_bias_decay",), decoder=True, bias_decay=True),
    "masked_untied": EngineSignature(SCE_UNTIED, "encoder", _SAE_LOSSES, decoder=True),
    "topk": EngineSignature(SCE_TOPK, "dict", ("loss",), norm_floor=0.0, topk=True),
    "tied_learned_center": EngineSignature(SCE_TIED_LEARNED_CENTER, "encoder", _SAE_LOSSES, learned_center=True),
    # FunctionalPositiveTiedSAE encodes and reconstructs x + 0.18 (autoencoders/mlp_tests.py:104, :110)
    "positive_tied": EngineSignature(SCE_TIED, "encoder", _SAE_LOSSES + ("l_bias_decay",), bias_decay=True,
                                     encoder_nonneg=True, input_shift=0.18),
    # forward-only kinds of metrics.evaluate_dicts / top_activating_fragments (no DictSignature trains them):
    # RandomDict decodes with its raw rows, ICAEncoder's code is signed and linear
    "random": EngineSignature(SCE_UNTIED, "encoder", _SAE_LOSSES, decoder=True, decoder_raw=True),
    "ica": EngineSignature(SCE_UNTIED, "encoder", _SAE_LOSSES, decoder=True, code_linear=True),
}


def plan_structs(sig: EngineSignature, params, buffers, mu, nu, *, batch_max: int, x_per_model: bool, centering: int,
                 adam: AdamConfig, adam_count_mode: str, fwd_passes: int, bwd_passes: int, arith: str):
    """``(SceDesc, SceBuffers, keep)`` of a plan of ``sig`` over the stacked ``params`` / ``buffers`` and the Adam moments
    ``mu`` / ``nu`` (keyed like ``params``); a ``coef_mask`` in ``buffers`` is applied whatever the signature (padding
    rows). ``keep`` holds the buffers as the engine reads them, by name; it and the tensors passed must outlive the plan.
    Reads only ``data_ptr()``: no CUDA call."""
    keep = {}

    def converted(name, dtype):
        if name not in buffers:
            return None
        keep[name] = buffers[name].to(dtype=dtype).contiguous()
        return keep[name].data_ptr()

    def param(name):   # a parameter and its Adam moments
        return params[name].data_ptr(), mu[name].data_ptr(), nu[name].data_ptr()

    main = params[sig.main]
    modifiers = (SCE_CODE_LINEAR if sig.code_linear else 0) | (SCE_DECODER_RAW if sig.decoder_raw else 0)
    desc = SceDesc(
        variant=sig.variant | modifiers, n_models=main.shape[0], d=main.shape[2], n=main.shape[1], batch_max=batch_max,
        x_per_model=int(x_per_model), lr=adam.lr, beta1=adam.b1, beta2=adam.b2, eps=adam.eps, eps_root=adam.eps_root,
        adam_count_mode=SCE_ADAM_FROZEN_T1 if adam_count_mode == "frozen_t1" else SCE_ADAM_STANDARD,
        fwd_passes=fwd_passes, bwd_passes=bwd_passes, norm_floor=sig.norm_floor, arith=arith_code(arith),
        centering=centering, encoder_nonneg=int(sig.encoder_nonneg), input_shift=sig.input_shift)
    bufs = SceBuffers()
    bufs.encoder, bufs.encoder_m, bufs.encoder_v = param(sig.main)
    if sig.topk:
        bufs.sparsity = converted("sparsity", torch.int64)
        desc.topk_k_max = int(keep["sparsity"].max())
    else:
        bufs.encoder_bias, bufs.bias_m, bufs.bias_v = param("encoder_bias")
        bufs.l1_alpha = converted("l1_alpha", torch.float32)
        if sig.bias_decay:
            bufs.bias_decay = converted("bias_decay", torch.float32)
    if sig.decoder:
        bufs.decoder, bufs.decoder_m, bufs.decoder_v = param("decoder")
    if sig.learned_center:
        bufs.center, bufs.center_m, bufs.center_v = param("center")
    bufs.coef_mask = converted("coef_mask", torch.uint8)
    if centering:
        # FunctionalTiedSAE.center (sae_ensemble.py:126-128) runs on the device: (x - trans) planes, GEMM with rot, * scale
        bufs.center_trans, bufs.center_rot, bufs.center_scale = (converted(k, torch.float32) for k in
                                                                 ("center_trans", "center_rot", "center_scale"))
    return desc, bufs, keep


class SceError(RuntimeError):
    pass


_lib = None


def load():
    """Load libsce.so once; raise loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SceError(
            f"{LIB_PATH} not found: the CUDA engine has not been built. Run `make` at the repository root "
            "(or `python -c 'import __graft_entry__ as g; g.build()'`). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, i, ll = C.c_void_p, C.c_int, C.c_longlong
    lib.sce_version.restype = i
    lib.sce_last_error.restype = C.c_char_p
    lib.sce_workspace_bytes.restype = C.c_size_t
    lib.sce_workspace_bytes.argtypes = [C.POINTER(SceDesc)]
    lib.sce_plan_create.argtypes = [C.POINTER(SceDesc), C.POINTER(SceBuffers), C.POINTER(vp)]
    lib.sce_plan_destroy.argtypes = [vp]
    lib.sce_prepare.argtypes = [vp, vp]
    lib.sce_step.argtypes = [vp, vp, i, vp, vp, vp]
    lib.sce_step_host.argtypes = [vp, vp, i, vp, vp, vp]
    lib.sce_forward.argtypes = [vp, vp, i, vp, vp, vp, vp]
    lib.sce_read_code.argtypes = [vp, i, vp, vp]
    lib.sce_grads.argtypes = [vp, vp, i, vp, vp, vp, vp, vp, vp]
    lib.sce_read_center_grad.argtypes = [vp, vp, vp]
    lib.sce_gather_rows.argtypes = [vp, i, ll, i, vp, i, vp, vp, vp]
    lib.sce_last_launch_count.argtypes = [vp]
    lib.sce_get_step_count.argtypes = [vp]
    lib.sce_get_step_count.restype = ll
    lib.sce_set_step_count.argtypes = [vp, ll]
    lib.sce_profile_begin.argtypes = [vp]
    lib.sce_profile_end.argtypes = [vp, vp, vp]
    lib.sce_plan_arith.argtypes = [vp]
    lib.sce_input_absmax.argtypes = [vp, vp, vp]
    lib.sce_health.argtypes = [vp, vp, vp, vp]
    lib.sce_clear_health.argtypes = [vp, vp]
    lib.sce_active_counts.argtypes = [vp, i, vp, vp]
    lib.sce_similarity_workspace_bytes.restype = C.c_size_t
    lib.sce_similarity_workspace_bytes.argtypes = [i, i, i, i, i, i, i]
    f = C.c_float
    lib.sce_similarity.argtypes = [vp, i, i, vp, f, i, vp, i, i, vp, f, i, i, vp, i, i, vp, vp, vp, vp, C.c_size_t, vp]
    lib.sce_forward_stats_workspace_bytes.restype = C.c_size_t
    lib.sce_forward_stats_workspace_bytes.argtypes = [C.POINTER(SceDesc), i]
    lib.sce_forward_stats.argtypes = [vp, vp, i, i, i, vp, vp, vp, vp, vp, vp, vp, C.c_size_t, vp]
    lib.sce_fragments_workspace_bytes.restype = C.c_size_t
    lib.sce_fragments_workspace_bytes.argtypes = [C.POINTER(SceDesc), i, i]
    lib.sce_forward_fragments.argtypes = [vp, vp, i, i, ll, i, i, C.c_ulonglong, vp, vp, vp, vp, vp, vp, vp, vp,
                                          C.c_size_t, vp]
    lib.sce_forward_split_workspace_bytes.restype = C.c_size_t
    lib.sce_forward_split_workspace_bytes.argtypes = [C.POINTER(SceDesc), i, i]
    lib.sce_forward_split.argtypes = [vp, vp, i, i, vp, vp, vp, vp, vp, vp, C.c_size_t, vp]
    lib.sce_interference_workspace_bytes.restype = C.c_size_t
    lib.sce_interference_workspace_bytes.argtypes = [C.POINTER(SceDesc), i]
    lib.sce_code_interference.argtypes = [vp, i, vp, vp, vp, C.c_size_t, vp]
    lib.sce_expected_interference_workspace_bytes.restype = C.c_size_t
    lib.sce_expected_interference_workspace_bytes.argtypes = [i, i, i]
    lib.sce_expected_interference.argtypes = [vp, i, i, vp, i, vp, vp, vp, C.c_size_t, vp]
    lib.sce_cross_moments_workspace_bytes.restype = C.c_size_t
    lib.sce_cross_moments_workspace_bytes.argtypes = [vp, vp, i]
    lib.sce_cross_moments.argtypes = [vp, vp, i, vp, vp, C.c_size_t, vp]
    lib.sce_correlation_finish.argtypes = [vp, i, i, i, vp, vp, ll, vp, vp, vp, vp, vp, vp, vp]
    lib.sce_synth_rows.argtypes = [vp, i, i, vp, i, ll, i, C.c_ulonglong, i, f, vp, i, vp, vp, vp, i, vp]
    lib.sce_second_moments_workspace_bytes.restype = C.c_size_t
    lib.sce_second_moments_workspace_bytes.argtypes = [i, i]
    lib.sce_second_moments.argtypes = [vp, i, i, i, vp, i, vp, vp, vp, vp, C.c_size_t, vp]
    lib.sce_ica_pass_workspace_bytes.restype = C.c_size_t
    lib.sce_ica_pass_workspace_bytes.argtypes = [i, i, i]
    lib.sce_ica_pass.argtypes = [vp, i, i, i, vp, vp, i, f, i, vp, vp, vp, vp, C.c_size_t, vp]
    lib.sce_nmf_project_workspace_bytes.restype = C.c_size_t
    lib.sce_nmf_project_workspace_bytes.argtypes = [i, i, i]
    lib.sce_nmf_project.argtypes = [vp, i, i, i, vp, vp, i, i, vp, vp, vp, vp, C.c_size_t, vp]
    lib.sce_nmf_grams_workspace_bytes.restype = C.c_size_t
    lib.sce_nmf_grams_workspace_bytes.argtypes = [i, i, i]
    lib.sce_nmf_grams.argtypes = [vp, i, i, i, vp, vp, i, i, vp, vp, vp, vp, C.c_size_t, vp]
    lib.sce_nmf_residual_workspace_bytes.restype = C.c_size_t
    lib.sce_nmf_residual_workspace_bytes.argtypes = [i, i]
    lib.sce_nmf_residual.argtypes = [vp, i, i, i, vp, vp, i, vp, vp, vp, C.c_size_t, vp]
    lib.sce_nmf_cd_sweep_workspace_bytes.restype = C.c_size_t
    lib.sce_nmf_cd_sweep_workspace_bytes.argtypes = [i, i]
    lib.sce_nmf_cd_sweep.argtypes = [vp, i, i, i, vp, vp, i, C.c_double, vp, vp, vp, C.c_size_t, vp]
    lib.sce_track_workspace_bytes.restype = C.c_size_t
    lib.sce_track_workspace_bytes.argtypes = [C.POINTER(SceDesc), i]
    lib.sce_step_tracked.argtypes = [vp, vp, i, vp, vp, C.POINTER(SceTrack), vp]
    lib.sce_resample.argtypes = [vp, C.POINTER(SceTrack), f, vp, vp, vp, vp]
    for name in EXPORTS:
        getattr(lib, name)  # AttributeError here means header and library disagree
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().sce_last_error().decode("utf-8", "replace")
        raise SceError(f"{what} failed (status {rc}): {msg}")


def arith_code(name: str) -> int:
    """The sce_arith code of "auto", "bf16x3" or "f16f8"."""
    if name not in ARITH_CODE:
        raise ValueError(f"arith must be one of {sorted(ARITH_CODE)}, got {name!r}")
    return ARITH_CODE[name]


def workspace(nbytes: int, device, what: str):
    """(tensor, address): ``nbytes`` of device memory at the 1024-byte aligned address every libsce workspace needs.
    ``nbytes`` comes from one of the size queries, which return 0 for arguments they reject (``what`` names it)."""
    if nbytes == 0:
        check(-1, what)
    ws = torch.empty(nbytes + 1024, dtype=torch.uint8, device=device)
    return ws, (ws.data_ptr() + 1023) // 1024 * 1024


def create_plan(desc: SceDesc, bufs: SceBuffers, device):
    """sce_plan_create with a workspace of the size ``desc`` needs, allocated on ``device`` and set in ``bufs``:
    (plan, workspace tensor). The tensor must outlive the plan."""
    lib = load()
    nbytes = lib.sce_workspace_bytes(C.byref(desc))
    ws, bufs.workspace = workspace(nbytes, device, "sce_workspace_bytes")
    bufs.workspace_bytes = nbytes
    plan = C.c_void_p()
    check(lib.sce_plan_create(C.byref(desc), C.byref(bufs), C.byref(plan)), "sce_plan_create")
    return plan, ws
