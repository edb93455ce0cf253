"""GPU tests of the callers either side of the step (SURVEY §8 f1/f2): device-side batch gather, the drop-in
``ensemble_train_loop``, chunk streaming + checkpoint layout, resume, per-model batches, the host-fed C-ABI step."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from engine_cases import clone_models, relnorm
from oracle import sae_oracle as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_gather_rows_bit_exact(dtype):
    """out[r] = float32(chunk[idx[r]]) - sub is pure data movement + one subtraction: bit-exact vs torch."""
    from sparse_coding_b200.train_loop import gather_rows
    gen = torch.Generator().manual_seed(0)
    chunk = torch.randn(5000, 192, generator=gen).to(dtype)
    idx = torch.randint(0, 5000, (777,), generator=gen)
    sub = torch.randn(192, generator=gen)
    dev = chunk.cuda()
    assert torch.equal(gather_rows(dev, idx.cuda()).cpu(), chunk[idx].float())
    assert torch.equal(gather_rows(dev, idx.cuda(), sub=sub.cuda()).cpu(), chunk[idx].float() - sub)
    assert torch.equal(gather_rows(dev, None).cpu(), chunk.float())
    assert gather_rows(dev, idx[:1].cuda()).shape == (1, 192)


def test_ensemble_train_loop_matches_reference_loop():
    """big_sweep.py:159-199 semantics on one chunk: same seeds, same sampler, same batches (incl. the short last
    one) as the restated reference loop; final parameters agree with the oracle trained on the same batches."""
    import sparse_coding_b200 as S
    from sparse_coding_b200.train_loop import ensemble_train_loop
    torch.manual_seed(0)
    d, n, N, B = 64, 128, 1000, 256
    models = [S.FunctionalTiedSAE.init(d, n, a) for a in (1e-3, 1e-2)]
    chunk = torch.randn(N, d, generator=torch.Generator().manual_seed(5)).half()      # chunks are fp16 on disk
    ens = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    ref = O.RefPortEnsemble(clone_models(models), O.SIG_LOSSES["tied"], lr=1e-3)

    class Cfg:
        use_wandb = False

    class Counter:
        value = -1

    mk = lambda: torch.utils.data.BatchSampler(torch.utils.data.RandomSampler(range(N)), batch_size=B, drop_last=False)
    ctr = Counter()
    ensemble_train_loop(ens, Cfg(), {"device": "cuda", "batch_size": B}, "ens", mk(), chunk, ctr)
    assert ctr.value == 3                                     # 4 batches: 256, 256, 256, 232
    torch.manual_seed(0)                                      # what the reference loop does at entry
    np.random.seed(0)
    data = chunk.float()
    for idxs in mk():
        ref.step_batch(data[idxs])
    assert relnorm(ens.params["encoder"], ref.params["encoder"]) <= 1e-3
    assert relnorm(ens.params["encoder_bias"], ref.params["encoder_bias"]) <= 1e-3 + 1e-9


def test_wandb_logging_keys():
    import sparse_coding_b200 as S
    from sparse_coding_b200.train_loop import ensemble_train_loop
    logs = []

    class Run:
        def log(self, d, commit=True):
            logs.append(d)

    class Cfg:
        use_wandb = True
        wandb_instance = Run()
        ensemble_hyperparams = ["dict_size"]
        buffer_hyperparams = ["l1_alpha"]

    class Counter:
        value = 0

    torch.manual_seed(0)
    models = [S.FunctionalTiedSAE.init(32, 64, a) for a in (1e-3, 1e-2)]
    ens = S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    sampler = torch.utils.data.BatchSampler(torch.utils.data.SequentialSampler(range(128)), batch_size=64, drop_last=False)
    ensemble_train_loop(ens, Cfg(), {"device": "cuda", "dict_size": 64}, "e0", sampler, torch.randn(128, 32), Counter())
    assert len(logs) == 2
    keys = set(logs[0])
    for l1 in ("1.00E-03", "1.00E-02"):
        for k in ("loss", "l_reconstruction", "l_l1", "num_nonzero"):
            assert f"e0_dict_size_64_l1_alpha_{l1}_{k}" in keys
    assert all(isinstance(v, float) for v in logs[0].values())


def test_chunk_streaming_checkpoints_and_resume(tmp_path):
    """{i}.pt fp16 chunks -> streamed training -> `_{i}/learned_dicts.pt` in the reference's pickle layout; a
    resumed ensemble (params + Adam moments + step count) continues bit-identically."""
    import sparse_coding_b200 as S
    from sparse_coding_b200.train_loop import load_resume_state, save_resume_state, train_on_chunks
    data = tmp_path / "data"
    out = tmp_path / "out"
    data.mkdir()
    gen = torch.Generator().manual_seed(0)
    for i in range(3):
        torch.save(torch.randn(700, 64, generator=gen).half(), data / f"{i}.pt")
    torch.manual_seed(1)
    models = [S.FunctionalTiedSAE.init(64, 128, a) for a in (1e-3, 1e-2)]
    args = {"device": "cuda", "dict_size": 128, "batch_size": 256}
    mk = lambda: S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda",
                                      adam_count_mode="standard")
    ens = mk()
    dicts = train_on_chunks(ens, args, str(data), str(out), 256, ["dict_size"], ["l1_alpha"], chunk_order=[0, 1, 2],
                            center_activations=True)
    assert os.path.exists(out / "_2" / "learned_dicts.pt") and os.path.exists(out / "means.pt")
    loaded = torch.load(out / "_2" / "learned_dicts.pt", weights_only=False)
    assert len(loaded) == 2 and type(loaded[0][0]).__module__ == "autoencoders.learned_dict"
    assert loaded[1][1] == {"dict_size": 128, "l1_alpha": pytest.approx(1e-2)}
    torch.testing.assert_close(loaded[0][0].encoder, ens.params["encoder"][0].cpu())
    x = torch.randn(16, 64)
    assert loaded[0][0].predict(x).shape == (16, 64)
    # --- resume: train 2 chunks, save, reload, train the third == training 3 chunks in one go
    ens_a = mk()
    train_on_chunks(ens_a, args, str(data), str(tmp_path / "o2"), 256, ["dict_size"], ["l1_alpha"], chunk_order=[0, 1])
    save_resume_state(ens_a, str(tmp_path / "resume.pt"))
    ens_b = load_resume_state(str(tmp_path / "resume.pt"), "cuda")
    assert ens_b._steps == 6 and ens_b.adam_count_mode == "standard"
    train_on_chunks(ens_b, args, str(data), str(tmp_path / "o3"), 256, ["dict_size"], ["l1_alpha"], chunk_order=[2])
    ens_c = mk()
    train_on_chunks(ens_c, args, str(data), str(tmp_path / "o4"), 256, ["dict_size"], ["l1_alpha"], chunk_order=[0, 1, 2])
    assert torch.equal(ens_b.params["encoder"], ens_c.params["encoder"])
    assert torch.equal(ens_b.optim_states["nu"]["encoder"], ens_c.optim_states["nu"]["encoder"])


def test_per_model_batches_expand_dims_false():
    """step_batch(x, expand_dims=False) with x [M,B,d] (ensemble.py:177-178): every model sees its own batch."""
    import sparse_coding_b200 as S
    torch.manual_seed(0)
    d, n, B = 64, 128, 96
    models = [S.FunctionalSAE.init(d, n, a) for a in (1e-3, 1e-2, 3e-2)]
    ens = S.FunctionalEnsemble(clone_models(models), S.FunctionalSAE, S.adam, {"lr": 1e-3}, device="cuda")
    X = torch.randn(3, B, d)
    grads, (loss, aux) = ens.grads_batch(X.cuda(), expand_dims=False)
    for i, (p, b) in enumerate(models):
        f = O.untied_grads(p["encoder"].double(), p["encoder_bias"].double(), p["decoder"].double(), X[i].double(),
                           float(b["l1_alpha"]))
        assert abs(float(loss["loss"][i]) - float(f["loss"])) <= 1e-4 * float(f["loss"])
        assert relnorm(grads["decoder"][i], f["grads"]["decoder"]) <= 2e-4
        assert relnorm(grads["encoder"][i], f["grads"]["encoder"]) <= 2e-4


def test_calc_grads_reference_shape():
    """ensemble.calc_grads(params, buffers, batch.expand(M, B, d)) as step_batch drives it in the reference
    (ensemble.py:177-180)."""
    import sparse_coding_b200 as S
    torch.manual_seed(0)
    models = [S.FunctionalTiedSAE.init(32, 64, a) for a in (1e-3, 1e-2)]
    ens = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    X = torch.randn(48, 32).cuda()
    g1, (l1, _) = ens.calc_grads(ens.params, ens.buffers, X.expand(2, 48, 32))
    g2, (l2, _) = ens.grads_batch(X)
    assert torch.equal(g1["encoder"], g2["encoder"]) and torch.equal(l1["loss"], l2["loss"])
    with pytest.raises(ValueError):
        ens.calc_grads({k: v.clone() for k, v in ens.params.items()}, ens.buffers, X.expand(2, 48, 32))


def test_host_fed_step_through_c_abi():
    """sce_step_host: HOST batch in, HOST losses out (the e2e path of bench.py), identical to the device path."""
    import sparse_coding_b200 as S
    from sparse_coding_b200 import _lib
    torch.manual_seed(0)
    d, n, B = 64, 128, 200
    models = [S.FunctionalTiedSAE.init(d, n, a) for a in (1e-3, 1e-2)]
    ens_a = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    ens_b = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    X = torch.randn(B, d).pin_memory()
    la, _ = ens_a.step_batch(X.cuda())
    ens_b.forward_batch(X.cuda())                       # builds the plan
    losses = torch.empty(2, 4).pin_memory()
    nnz = torch.empty(2).pin_memory()
    lib = _lib.load()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.sce_step_host(ens_b._plan, X.data_ptr(), B, losses.data_ptr(), nnz.data_ptr(), stream), "sce_step_host")
    assert torch.equal(losses[:, 0], la["loss"].cpu())
    assert torch.equal(ens_a.params["encoder"], ens_b.params["encoder"])
    assert lib.sce_get_step_count(ens_b._plan) == 1


def test_on_device_evaluation_matches_learned_dict_metrics():
    """metrics.evaluate (one fused forward for all models) == FVU / mean L0 / ever-active computed the reference's
    way from the exported LearnedDicts (standard_metrics.py:305-314, 446-454)."""
    import sparse_coding_b200 as S
    from sparse_coding_b200.metrics import evaluate
    torch.manual_seed(0)
    d, n = 64, 256
    models = [S.FunctionalTiedSAE.init(d, n, a) for a in (1e-3, 1e-2)]
    ens = S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    gen = torch.Generator().manual_seed(3)
    for _ in range(20):
        ens.step_batch(torch.randn(256, d, generator=gen).cuda())
    held = torch.randn(1000, d, generator=gen)
    got = evaluate(ens, held.cuda(), n_ever_active=True)
    for i, (p, b) in enumerate(ens.unstack(device="cpu")):
        ld = S.FunctionalTiedSAE.to_learned_dict(p, b)
        c = ld.encode(ld.center(held))
        assert abs(float(got["fvu"][i]) - float(O.fvu(held, ld.predict(held)))) <= 1e-4 * float(got["fvu"][i]) + 1e-6
        assert abs(float(got["mean_l0"][i]) - float((c != 0).float().sum(-1).mean())) <= 0.02
        assert abs(int(got["n_ever_active"][i]) - int((c != 0).any(0).sum())) <= 1


def _child_steps(state_dict, batches, done):
    """Body of a reference-style worker process (cluster_runs.py:15-36 `job_wrapper`): rebuild the ensemble from
    its state_dict (device tensors arrive through CUDA IPC) and train on the parent's memory in place."""
    import sparse_coding_b200 as S
    torch.set_grad_enabled(False)
    ens = S.FunctionalEnsemble.from_state(state_dict)
    for x in batches:
        ens.step_batch(x.to(ens.device))
    torch.cuda.synchronize()
    done.value = 1


def test_spawned_worker_trains_parent_memory_in_place():
    """The reference dispatches every chunk to a freshly spawned process per ensemble and relies on the child
    mutating the parent's device tensors through CUDA IPC (cluster_runs.py:100-157, ensemble.py:125-161). The
    engine-backed ensemble must survive that round trip: state_dict() pickles, from_state() in the child builds its
    own plan/workspace, and parameters + Adam moments change in the parent."""
    import torch.multiprocessing as mp
    import sparse_coding_b200 as S
    torch.manual_seed(0)
    d, n, B = 64, 128, 256
    models = [S.FunctionalTiedSAE.init(d, n, a) for a in (1e-3, 1e-2)]
    ens = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda:0")
    twin = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda:0")
    gen = torch.Generator().manual_seed(1)
    batches = [torch.randn(B, d, generator=gen) for _ in range(3)]
    before = ens.params["encoder"].clone()
    ens.to_shared_memory()
    ctx = mp.get_context("spawn")
    done = ctx.Value("i", 0)
    proc = ctx.Process(target=_child_steps, args=(ens.state_dict(), batches, done))
    proc.start()
    proc.join(timeout=300)
    assert proc.exitcode == 0 and done.value == 1
    for x in batches:
        twin.step_batch(x.cuda())
    torch.cuda.synchronize()
    assert not torch.equal(ens.params["encoder"], before)
    assert torch.equal(ens.params["encoder"], twin.params["encoder"])
    assert torch.equal(ens.optim_states["nu"]["encoder_bias"], twin.optim_states["nu"]["encoder_bias"])


def test_two_devices_in_one_process():
    """Plans on different GPUs of one process (the reference builds one ensemble per device in the parent,
    big_sweep_experiments.py:265-291). Skipped on single-GPU boxes."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import sparse_coding_b200 as S
    torch.manual_seed(0)
    models = [S.FunctionalTiedSAE.init(64, 128, a) for a in (1e-3, 1e-2)]
    X = torch.randn(256, 64)
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        ens = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device=dev)
        loss, _ = ens.step_batch(X.to(dev))
        outs.append((loss["loss"].cpu(), ens.params["encoder"].cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_c_abi_error_paths_on_device():
    """Errors cross the ABI as negative status + thread-local message, never as a crash: wrong device class of
    arguments, batch larger than the plan, misaligned / short workspace."""
    import sparse_coding_b200 as S
    from sparse_coding_b200 import _lib
    lib = _lib.load()
    torch.manual_seed(0)
    models = [S.FunctionalTiedSAE.init(32, 64, 1e-3)]
    ens = S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    ens.step_batch(torch.randn(128, 32).cuda())                       # plan for batch_max = 128
    x = torch.randn(256, 32).cuda()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.sce_step(ens._plan, x.data_ptr(), 256, None, None, stream) == -1
    assert b"batch_max" in lib.sce_last_error()
    assert lib.sce_step(ens._plan, None, 64, None, None, stream) == -1
    assert lib.sce_read_code(ens._plan, 0, x.data_ptr(), stream) == -1
    # the Python layer re-plans transparently for a larger batch
    loss, _ = ens.step_batch(x)
    assert torch.isfinite(loss["loss"]).all()
    # short / misaligned workspace
    desc = _lib.SceDesc(variant=0, n_models=1, d=32, n=64, batch_max=128, x_per_model=0, lr=1e-3, beta1=0.9, beta2=0.999,
                        eps=1e-8, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-8)
    need = lib.sce_workspace_bytes(C.byref(desc))
    ws = torch.empty(need + 2048, dtype=torch.uint8, device="cuda")
    p = ens.params
    mu, nu = ens.optim_states["mu"], ens.optim_states["nu"]
    bufs = _lib.SceBuffers(encoder=p["encoder"].data_ptr(), encoder_bias=p["encoder_bias"].data_ptr(),
                           encoder_m=mu["encoder"].data_ptr(), encoder_v=nu["encoder"].data_ptr(),
                           bias_m=mu["encoder_bias"].data_ptr(), bias_v=nu["encoder_bias"].data_ptr(),
                           workspace=(ws.data_ptr() + 1023) // 1024 * 1024 + 16, workspace_bytes=need)
    plan = C.c_void_p()
    assert lib.sce_plan_create(C.byref(desc), C.byref(bufs), C.byref(plan)) == -3 and b"aligned" in lib.sce_last_error()
    bufs.workspace = (ws.data_ptr() + 1023) // 1024 * 1024
    bufs.workspace_bytes = need - 1
    assert lib.sce_plan_create(C.byref(desc), C.byref(bufs), C.byref(plan)) == -3 and b"too small" in lib.sce_last_error()
    bufs.workspace_bytes = need
    assert lib.sce_plan_create(C.byref(desc), C.byref(bufs), C.byref(plan)) == 0
    assert lib.sce_plan_destroy(plan) == 0
    # top-k: sce_prepare reads the sparsities; k outside [1, n], or above topk_k_max where the plan keeps lists (1..256),
    # is rejected before any selection could write past its lists. The valid ones (positive controls) prepare.
    d, n = 32, 256
    dct = torch.randn(1, n, d, device="cuda")
    mom = torch.zeros_like(dct)
    for k, k_max, want in ((20, 16, b"topk_k_max"), (0, 16, b"outside [1, n"), (n + 1, 0, b"outside [1, n"),
                           (300, 300, b"outside [1, n"), (16, 16, None), (9, 16, None), (20, 0, None), (n, 300, None)):
        desc = _lib.SceDesc(variant=_lib.SCE_TOPK, n_models=1, d=d, n=n, batch_max=16, x_per_model=0, lr=0.0, beta1=0.9,
                            beta2=0.999, eps=1e-8, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3,
                            norm_floor=0.0, arith=0, topk_k_max=k_max, centering=0)
        sp = torch.tensor([k], dtype=torch.int64, device="cuda")
        bufs = _lib.SceBuffers(encoder=dct.data_ptr(), encoder_m=mom.data_ptr(), encoder_v=mom.data_ptr(),
                               sparsity=sp.data_ptr())
        plan, ws = _lib.create_plan(desc, bufs, torch.device("cuda"))
        try:
            if want is None:
                assert lib.sce_prepare(plan, stream) == 0, (k, k_max, lib.sce_last_error())
            else:
                assert lib.sce_prepare(plan, stream) == -1, (k, k_max)
                assert want in lib.sce_last_error(), (k, k_max, lib.sce_last_error())
        finally:
            lib.sce_plan_destroy(plan)
