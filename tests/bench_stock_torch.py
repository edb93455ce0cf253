"""Informational comparator (not a test, not the product): the restated reference step — stock PyTorch ops under
vmap(grad(loss)) + Adam, i.e. what HoagyC/sparse_coding would launch on a GPU — timed on the GPU at BASELINE
config 2, in true fp32 (the reference never enables TF32) and with TF32 allowed. Lives under tests/ because it
drives the oracle.   python tests/bench_stock_torch.py"""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from oracle import sae_oracle as O
import sparse_coding_b200 as S

M, d, n, B = 16, 512, 4096, 8192
dev = torch.device("cuda", 0)
out = {"workload": "cfg2: 16 TiedSAE d=512 n=4096 batch=8192, one step = vmap(grad(loss)) + Adam on stock PyTorch ops"}
for name, tf32 in (("fp32", False), ("tf32", True)):
    torch.backends.cuda.matmul.allow_tf32 = tf32
    torch.backends.cudnn.allow_tf32 = tf32
    torch.manual_seed(0)
    models = [S.FunctionalTiedSAE.init(d, n, float(a)) for a in np.logspace(-4, -2, M)]
    models = [({k: v.to(dev) for k, v in p.items()}, {k: v.to(dev) for k, v in b.items()}) for p, b in models]
    ens = O.RefPortEnsemble(models, O.SIG_LOSSES["tied"], lr=1e-3)
    x = torch.randn(B, d, device=dev)
    for _ in range(3):
        ens.step_batch(x)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    K = 10
    e0.record()
    for _ in range(K):
        loss, aux = ens.step_batch(x)
        nnz = aux["c"].count_nonzero(dim=-1).float().mean(dim=-1)     # big_sweep.py:171
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    out[name] = {"ms_per_step": ms, "activations_per_s": B / (ms * 1e-3),
                 "peak_mem_gb": torch.cuda.max_memory_allocated() / 2**30}
    del ens, models
    torch.cuda.empty_cache()
print(json.dumps(out))
