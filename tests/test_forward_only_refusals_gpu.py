"""The two rules every forward-only pass of a plan shares, on the GPU:
  evaluable   a non-negative tied plan on a shifted input (its export, a TiedSAE, has another forward) is refused by
              sce_forward_stats, sce_forward_fragments, sce_forward_split, sce_code_interference and sce_cross_moments
              (on either side) with rc -1 and one message, and every workspace query returns 0 for it
  last call   after a training step of a dense f16f8 plan whose weight gradient runs on native E5M2 wgmma (the step
              leaves the code's residual plane batch-major only), sce_code_interference and sce_cross_moments (either
              side) refuse and leave their accumulators bitwise untouched; a following sce_forward_stats makes both run
All these refusals are made on the host, before any launch."""
import ctypes as C

import pytest
import torch

import engine_cases as EC
from oracle.plan_paths import launch_bound
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT

pytestmark = pytest.mark.gpu
DEV = EC.DEV
NOT_EVALUABLE = ("not available for the learned-centre variant or with encoder_nonneg / input_shift; evaluate the "
                 "exported dictionaries (TiedSAE)")
TRAINING_STEP = "a plan's last call was a training step; follow sce_forward_stats"


def stats_plan(n, d, batch_max, arith, seed):
    """A _StatsPlan of one TiedSAE, evaluable, and the rows of one forward pass it has run."""
    ld = EC.tied(n, d, seed)
    p = MT._StatsPlan(EC.one_key([ld], arith), [ld], batch_max, arith, DEV)
    p.stats(EC.synth(batch_max, d, seed), 1, 0)
    return p


def interference(lib, plan, desc, B, cap, nz):
    need = lib.sce_interference_workspace_bytes(C.byref(desc), B)
    ws, ptr = _lib.workspace(need, DEV, "sce_interference_workspace_bytes")
    rc = lib.sce_code_interference(plan, B, cap.data_ptr(), nz.data_ptr(), ptr, need, None)
    return rc, lib.sce_last_error().decode()


def cross(lib, a, b, B, acc):
    need = lib.sce_cross_moments_workspace_bytes(a, b, B)
    ws, ptr = _lib.workspace(need, DEV, "sce_cross_moments_workspace_bytes")
    rc = lib.sce_cross_moments(a, b, B, acc.data_ptr(), ptr, need, None)
    return rc, lib.sce_last_error().decode()


def test_not_evaluable_plan():
    lib = _lib.load()
    M, d, n, B = 2, 64, 128, 64
    models, sig = EC.make_models("positive_tied", M, d, n, 3)
    with torch.cuda.device(DEV):
        ens = EC.ensemble(models, sig, "bf16x3")
        x = EC.synth(B, d, 4)
        ens.forward_batch(x)
        p, desc = ens._plan, ens._plan_desc
        assert desc.encoder_nonneg and desc.input_shift != 0.0
        good = stats_plan(n, d, B, "bf16x3", 5)
        try:
            plain = _lib.SceDesc.from_buffer_copy(desc)
            plain.encoder_nonneg, plain.input_shift = 0, 0.0
            for q in (desc, plain):       # the plain descriptor is the positive control
                sizes = [lib.sce_forward_stats_workspace_bytes(C.byref(q), B),
                         lib.sce_fragments_workspace_bytes(C.byref(q), B, 32),
                         lib.sce_forward_split_workspace_bytes(C.byref(q), B, 2),
                         lib.sce_interference_workspace_bytes(C.byref(q), B)]
                assert all(s == 0 for s in sizes) if q is desc else all(s > 0 for s in sizes), sizes
            assert lib.sce_cross_moments_workspace_bytes(p, good.plan, B) == 0
            assert lib.sce_cross_moments_workspace_bytes(good.plan, p, B) == 0
            assert lib.sce_cross_moments_workspace_bytes(good.plan, good.plan, B) > 0

            cap = torch.zeros(M, n, dtype=torch.float64, device=DEV)
            nz = torch.zeros(M, n, dtype=torch.int64, device=DEV)
            acc = torch.zeros(M * n * n, dtype=torch.float64, device=DEV)
            ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
            calls = {
                "forward_stats: ": lambda: lib.sce_forward_stats(p, x.data_ptr(), B, 1, 0, *([None] * 7), 0, None),
                "forward_fragments: ": lambda: lib.sce_forward_fragments(p, x.data_ptr(), B, 32, 0, 4, 0,
                                                                         C.c_ulonglong(0), *([None] * 8), 0, None),
                "forward_split: ": lambda: lib.sce_forward_split(p, x.data_ptr(), B, 2, ws.data_ptr(), *([None] * 4),
                                                                 None, 0, None),
                "code_interference: ": lambda: lib.sce_code_interference(p, B, cap.data_ptr(), nz.data_ptr(),
                                                                         ws.data_ptr(), ws.numel(), None),
                "cross_moments: plan_a: ": lambda: lib.sce_cross_moments(p, good.plan, B, acc.data_ptr(),
                                                                         ws.data_ptr(), ws.numel(), None),
                "cross_moments: plan_b: ": lambda: lib.sce_cross_moments(good.plan, p, B, acc.data_ptr(),
                                                                         ws.data_ptr(), ws.numel(), None),
            }
            for prefix, call in calls.items():
                rc = call()
                err = lib.sce_last_error().decode()
                assert rc == -1 and err == prefix + NOT_EVALUABLE, (prefix, rc, err)
            torch.cuda.synchronize()
            assert not cap.any() and not nz.any() and not acc.any()
        finally:
            good.close()


def test_code_after_a_training_step():
    lib = _lib.load()
    M, d, n, B = 4, 1024, 2048, 2048
    assert not launch_bound(M, B, n, d)         # the step's weight gradient runs from batch-major copies (dw_native)
    models, sig = EC.make_models("tied", M, d, n, 7)
    with torch.cuda.device(DEV):
        ens = EC.ensemble(models, sig, "f16f8")
        x = EC.batch(M, B, d, 8, False, True)
        ens.step_batch(x)
        assert ens.resolved_arith() == "f16f8"
        p, desc = ens._plan, ens._plan_desc
        other = stats_plan(64, 64, B, "f16f8", 9)    # the other side of the cross moments: evaluable, after a forward
        try:
            cap = torch.full((M, n), -7.0, dtype=torch.float64, device=DEV)
            nz = torch.full((M, n), -7, dtype=torch.int64, device=DEV)
            acc_ab = torch.full((M, 1, n, 64), -7.0, dtype=torch.float64, device=DEV)
            acc_ba = torch.full((1, M, 64, n), -7.0, dtype=torch.float64, device=DEV)
            results = {"code_interference: ": interference(lib, p, desc, B, cap, nz),
                       "cross_moments: plan_a: ": cross(lib, p, other.plan, B, acc_ab),
                       "cross_moments: plan_b: ": cross(lib, other.plan, p, B, acc_ba)}
            for prefix, (rc, err) in results.items():
                assert rc == -1 and err == prefix + TRAINING_STEP, (prefix, rc, err)
            torch.cuda.synchronize()
            for t in (cap, nz, acc_ab, acc_ba):
                assert bool((t == -7).all())

            # a forward pass of the plan's own: both calls read its code again
            need = lib.sce_forward_stats_workspace_bytes(C.byref(desc), B)
            ws, ptr = _lib.workspace(need, DEV, "sce_forward_stats_workspace_bytes")
            losses = torch.empty(M, _lib.SCE_LOSS_COLS, device=DEV)
            nnz = torch.empty(M, device=DEV)
            sums = torch.zeros(M, n, 4, dtype=torch.float64, device=DEV)
            counts = torch.zeros(M, n, dtype=torch.int32, device=DEV)
            _lib.check(lib.sce_forward_stats(p, x.data_ptr(), B, 1, 0, None, losses.data_ptr(), nnz.data_ptr(),
                                             sums.data_ptr(), counts.data_ptr(), None, ptr, need, None),
                       "sce_forward_stats")
            for prefix, (rc, err) in {"code_interference: ": interference(lib, p, desc, B, cap, nz),
                                      "cross_moments: plan_a: ": cross(lib, p, other.plan, B, acc_ab),
                                      "cross_moments: plan_b: ": cross(lib, other.plan, p, B, acc_ba)}.items():
                assert rc == 0, (prefix, err)
            torch.cuda.synchronize()
            assert 0 < int((nz + 7).sum()) <= int(counts.sum())     # the forward pass's active entries, counted
            for t in (cap, acc_ab, acc_ba):
                assert bool((t != -7).any())
        finally:
            other.close()
