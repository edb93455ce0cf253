"""Dead-feature resampling without a GPU: the fp64 oracle against the reference's own WorstIndices and replacement rule
(tests/golden/resample.pt, oracle/make_resample_golden.py), the argument checks of sce_track_workspace_bytes /
sce_step_tracked / sce_resample, the chunk schedule of train_on_chunks(resample_every=...), and the errors of the
Python API without a window or on the CPU."""
import ctypes as C
import os

import pytest
import torch

import sparse_coding_b200 as S
from oracle import resample_oracle as RO
from sparse_coding_b200 import _lib, train_loop

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resample.pt")


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


def test_window_order_matches_worst_indices(golden):
    g = golden["worst"]
    w = RO.Window(g["n_ndxs"], n=4, d=1)
    r0 = 0
    for B in g["batch_rows"]:
        e = g["losses"][r0:r0 + B]
        w.add(e, torch.arange(r0, r0 + B, dtype=torch.float32)[:, None], torch.zeros(B, 4))
        r0 += B
    assert r0 == g["losses"].numel()
    assert torch.equal(w.serial, g["get_worst"])                  # already in list order
    assert torch.equal(w.rows[:, 0].long(), g["get_worst"])       # each entry carries its own row


def test_replacement_matches_process_reinit(golden):
    g = golden["replace"]
    w = RO.Window(g["n_ndxs"], n=g["c_totals"].numel(), d=g["data"].shape[1])
    for r0 in range(0, 80, 24):                                    # any batching gives the same window
        rows = g["data"][r0:r0 + 24]
        w.add(g["losses"][r0:r0 + 24], rows, torch.zeros(rows.shape[0], g["c_totals"].numel()))
    counts = (g["c_totals"] != 0).long()
    dead = RO.dead_features(counts)
    assert torch.equal(dead, g["replace_ndxs"])
    out = RO.resample(g["encoder_before"].T, w.rows, dead, 0.2)
    want = g["encoder_after"].T.double()
    assert torch.equal(out["replaced"], dead)
    assert torch.allclose(out["W"], want, rtol=2e-7, atol=0)
    keep = torch.ones(want.shape[0], dtype=torch.bool)
    keep[dead] = False
    assert torch.equal(out["W"][keep].float(), g["encoder_before"].T[keep])


def test_oracle_leaves_extra_dead_features_and_skips_masked_padding():
    W = torch.randn(8, 4, dtype=torch.float64)
    counts = torch.tensor([0, 3, 0, 0, 1, 0, 0, 0])
    mask = torch.tensor([0, 0, 0, 0, 0, 0, 1, 1], dtype=torch.uint8)
    dead = RO.dead_features(counts, mask)
    assert dead.tolist() == [0, 2, 3, 5]
    rows = torch.randn(2, 4)
    out = RO.resample(W, rows, dead, 0.2, mask)
    assert out["replaced"].tolist() == [0, 2]
    assert torch.equal(out["W"][3], W[3]) and torch.equal(out["W"][6:], W[6:])
    mu = W[:6].norm(dim=-1).mean()
    assert torch.allclose(out["W"][2], rows[1].double() * 0.2 / mu)


def _desc(**kw):
    d = dict(variant=0, n_models=2, d=64, n=128, batch_max=256, x_per_model=0, lr=1e-3, beta1=0.9, beta2=0.999,
             eps=1e-8, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-8)
    d.update(kw)
    return _lib.SceDesc(**d)


def test_track_workspace_bytes():
    lib = _lib.load()
    desc = _desc()
    need = lib.sce_track_workspace_bytes(C.byref(desc), 128)
    assert need > 0 and need % 1024 == 0
    assert lib.sce_track_workspace_bytes(C.byref(desc), 16) < need
    desc.batch_max = 512
    assert lib.sce_track_workspace_bytes(C.byref(desc), 128) > need   # grows with the batch
    for bad in (0, -1, 129):
        assert lib.sce_track_workspace_bytes(C.byref(desc), bad) == 0
        assert b"n_worst" in lib.sce_last_error()
    desc.d = 63
    assert lib.sce_track_workspace_bytes(C.byref(desc), 16) == 0
    cfg2 = _desc(n_models=16, d=512, n=4096, batch_max=8192)
    assert lib.sce_track_workspace_bytes(C.byref(cfg2), 4096) < 16 * 2**20


@pytest.mark.parametrize("entry", ["step", "resample"])
def test_track_argument_errors_before_any_device_call(entry):
    lib = _lib.load()
    buf = (C.c_char * 8192)()
    base = (C.addressof(buf) + 1023) // 1024 * 1024

    def call(track, plan=None):
        if entry == "step":
            return lib.sce_step_tracked(plan, None, 1, None, None, track, None)
        return lib.sce_resample(plan, track, 0.2, None, None, None, None)

    def good():
        return _lib.SceTrack(err=base, serial=base, rows=base, filled=base, counts=base, next_serial=0, n_worst=4,
                             workspace=base, workspace_bytes=1024)

    assert call(None) == -1 and b"track is NULL" in lib.sce_last_error()
    for field in ("err", "serial", "rows", "filled", "counts"):
        t = good()
        setattr(t, field, None)
        assert call(C.byref(t)) == -1 and b"are required" in lib.sce_last_error(), field
    t = good()
    t.rows = base + 4
    assert call(C.byref(t)) == -1 and b"16-byte aligned" in lib.sce_last_error()
    t = good()
    t.n_worst = 0
    assert call(C.byref(t)) == -1 and b"n_worst" in lib.sce_last_error()
    t = good()
    assert call(C.byref(t)) == -1 and b"plan is NULL" in lib.sce_last_error()


class _FakeEnsemble:
    def __init__(self):
        self.calls = []
        self.n_models = 1

    def step_batch(self, batch):
        self.calls.append(("step", batch.shape[0]))

    def track_dead_features(self):
        self.calls.append(("track",))

    def resample_dead_features(self, ratio):
        self.calls.append(("resample", ratio))
        return {"n_dead": ratio}

    def stop_tracking(self):
        self.calls.append(("stop",))

    def unstack(self, device=None):
        return []


def _run(tmp_path, monkeypatch, n_chunks, **kw):
    monkeypatch.setattr(train_loop, "gather_rows", lambda chunk, idx, sub=None: chunk[idx])
    ens = _FakeEnsemble()
    chunks = [(10 + i, torch.zeros(5, 3)) for i in range(n_chunks)]
    train_loop.train_on_chunks(ens, {"device": "cpu"}, None, str(tmp_path), 2, [], [], chunks=chunks, **kw)
    return ens.calls


def test_chunk_schedule_of_train_on_chunks(tmp_path, monkeypatch):
    seen = []
    calls = _run(tmp_path, monkeypatch, 7, resample_every=3, resample_ratio=0.5,
                 on_resample=lambda i, idx, e, r: seen.append((i, idx, r["n_dead"])))
    assert seen == [(0, 10, 0.5), (3, 13, 0.5), (6, 16, 0.5)]
    kinds = [c[0] for c in calls]
    assert kinds.count("track") == 7 and kinds.count("step") == 7 * 3 and kinds[-1] == "stop"
    # a window opens before every chunk's first step; the resample follows that chunk's last step
    per_chunk = " ".join(kinds).split("track ")[1:]
    assert [("resample" in c) for c in per_chunk] == [i % 3 == 0 for i in range(7)]
    assert all(c.startswith("step step step") for c in per_chunk)


def test_no_resampling_calls_no_tracking_method(tmp_path, monkeypatch):
    calls = _run(tmp_path, monkeypatch, 4)
    assert {c[0] for c in calls} == {"step"}
    calls = _run(tmp_path, monkeypatch, 4, resample_every=0, on_resample=lambda *a: 1 / 0)
    assert {c[0] for c in calls} == {"step"}


def test_python_api_errors_without_window_and_on_cpu():
    models = [S.FunctionalTiedSAE.init(16, 32, 1e-3) for _ in range(2)]
    ens = S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cpu")
    with pytest.raises(RuntimeError, match="open window"):
        ens.resample_dead_features()
    with pytest.raises(RuntimeError, match="open window"):
        ens.worst_rows()
    with pytest.raises(RuntimeError, match="no CPU implementation"):
        ens.track_dead_features()
    assert "track" not in " ".join(ens.state_dict())
