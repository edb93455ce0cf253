#!/usr/bin/env python
"""Dictionary metrics on the engine against the reference's op sequence on the same GPU.
  mmcs_*: dictionary similarity (standard_metrics.py mmcs / mcs_duplicates / capacity_per_feature). One metric pass = the
          cosine maxima of every pair in both directions plus the capacity of every dictionary.
  eval_*: scores of exported dictionaries on activations (calc_moments_streaming + fraction_variance_unexplained +
          mean_nonzero_activations). One pass = metrics.evaluate_dicts of every dictionary over every row.
  interp_*: record selection for reading features (interpret.py make_feature_activation_dataset + interpret's choice of
          top and random records). One pass = metrics.top_activating_fragments of every dictionary over 50 000 fragments
          of 64 fp16 rows, 20 + 20 records per feature with their per-token values.
  topfvu_cfg2: the top- and rest-feature FVU (fraction_variance_unexplained_top_activating, n_top = 2) of the config-2
          dictionaries. One pass = metrics.evaluate_dicts(n_top=2), whose second pass is timed as the difference to the
          call without n_top.
  interference_cfg2: the expected interference (big_sweep.py calc_expected_interference) of the config-2 dictionaries.
          One pass = metrics.evaluate_dicts(interference=True); the difference to the call without it is the cost of the
          interference kernels.
  *_baselines: the same two passes on the baselines of sweep_baselines.py: one ICAEncoder, RandomDict(512) and
          IdentityReLU(512) at d = 512, in one pass (2^20 rows / 50 000 fragments of 64 rows).

    python tools/bench_metrics.py --workload mmcs_cfg2|mmcs_cfg5|eval_cfg2|eval_cfg5|interp_cfg2|interp_cfg5|
                                             eval_baselines|interp_baselines|topfvu_cfg2|
                                             interference_cfg2 [--steps K --warmup W --arith ...]

Prints one JSON line: CUDA-event ms per pass, algorithmic TFLOP/s (2 n_a n_b d per pair and per capacity), the same
computation as fp32 einsums + maxima and again with TF32 allowed, the maximum deviation of each from an fp64 result, and
the card name and power limit read in the same call. Writes nothing to disk."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def make_models(sig, M, d, n, seed):
    """M seeded TiedSAEs with L1 = logspace(-4, -2, M), as bench.py builds config 2."""
    torch.manual_seed(seed)
    return [sig.init(d, n, float(a)) for a in (np.logspace(-4, -2, M) if M > 1 else [1e-3])]


def setup(args):
    """(device, steps, warmup): cuda:0, made current, and the checked step counts."""
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_metrics.py needs a CUDA device (the engine has no CPU path)")
    if args.steps < 1:
        raise SystemExit("--steps must be at least 1")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    return dev, args.steps, max(args.warmup, 1)


def timed(fn, k, w):
    """(CUDA-event ms per call over k calls after w warm-up calls, the last result)."""
    for _ in range(w):
        r = fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(k):
        r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / k, r


def activations(N, d, dev):
    """[N, d] fp16 on dev: a sparse mixture of 2048 directions plus noise, seeded, generated in pieces of 2^16 rows."""
    gen = torch.Generator(device=dev).manual_seed(1)
    x = torch.empty(N, d, dtype=torch.float16, device=dev)
    for i in range(0, N, 1 << 16):
        k = min(1 << 16, N - i)
        feats = torch.nn.functional.normalize(torch.randn(2048, d, generator=gen, device=dev), dim=-1)
        code = (torch.rand(k, 2048, generator=gen, device=dev) < 0.01) * torch.rand(k, 2048, generator=gen, device=dev)
        x[i:i + k] = (code @ feats + 0.05 * torch.randn(k, d, generator=gen, device=dev)).half()
    return x


MMCS_WORKLOADS = {
    # name: (M, n, d, pairs, description)
    "mmcs_cfg2": (16, 4096, 512, "lower", "16 seeded config-2 TiedSAE dictionaries (4096 x 512): all 120 lower-triangle "
                                          "pairs, both directions, plus capacity of all 16"),
    "mmcs_cfg5": (2, 32768, 2048, [(1, 0)], "two config-5 TiedSAE dictionaries (32768 x 2048): one pair, both "
                                            "directions, plus capacity of each"),
}


def card_info(index):
    """(name, power limit in W) of the GPU, read in the same call as the measurement."""
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in r.stdout.strip().split(",")[:2]]
        return name, float(limit)
    except Exception:
        return torch.cuda.get_device_name(index), None


def run_mmcs(args):
    """Dictionary-similarity workloads (standard_metrics.py mmcs / mcs_duplicates / capacity_per_feature): one metric
    pass = the cosine maxima of every pair in both directions plus the capacity of every dictionary, on the engine and
    as the reference's op sequence (fp32 einsum + maxima per pair) on the same GPU, fp32 and TF32."""
    import sparse_coding_b200 as S
    from oracle import metrics_oracle as O
    from sparse_coding_b200 import metrics as MT

    dev, K, W = setup(args)
    M, n, d, pairs, desc = MMCS_WORKLOADS[args.workload]
    ens = S.FunctionalEnsemble(make_models(S.FunctionalTiedSAE, M, d, n, seed=0), S.FunctionalTiedSAE, S.adam,
                               {"lr": 1e-3}, device=dev)
    plist = [(i, j) for i in range(M) for j in range(i)] if pairs == "lower" else pairs

    def engine_pass():
        return MT.dictionary_similarity(ens, pairs=plist, arith=args.arith), MT.capacity(ens, arith=args.arith)

    ms, (res, cap) = timed(engine_pass, K, W)
    L = [ens.sig.to_learned_dict(p, b).get_learned_dict() for p, b in ens.unstack()]   # torch, fp32

    def stock_pass():
        rows, cols, caps = [], [], []
        for i, j in plist:
            s = torch.einsum("md,gd->mg", L[i], L[j])
            rows.append(s.max(dim=-1).values)
            cols.append(s.max(dim=0).values)
        for l in L:
            s = torch.einsum("md,nd->mn", l, l).pow(2)
            caps.append(torch.diag(s) / s.sum(dim=-1))
        return torch.stack(rows), torch.stack(cols), torch.stack(caps)

    k_ref = max(1, min(K, 3))
    tf32 = torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cuda.matmul.allow_tf32 = False
        ms_fp32, ref32 = timed(stock_pass, k_ref, 1)
        torch.backends.cuda.matmul.allow_tf32 = True
        ms_tf32, reftf = timed(stock_pass, k_ref, 1)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32

    # deviation of each from the fp64 result
    L64 = [l.double() for l in L]
    exact = [O.pair_maxima(L64[i], L64[j]) for i, j in plist]
    r64 = torch.stack([e[0] for e in exact])
    c64 = torch.stack([e[1] for e in exact])
    cap64 = torch.stack([O.capacity_blocked(l) for l in L64])

    def dev_of(rows, cols, caps):
        return {"cos_max_abs": float(max((rows.double() - r64).abs().max(), (cols.double() - c64).abs().max())),
                "capacity_max_rel": float(((caps.double() - cap64).abs() / cap64.abs()).max())}

    flops = 2.0 * n * n * d * (len(plist) + M)      # algorithmic: one [n, d] x [d, n] product per pair and per capacity
    name, limit = card_info(0)
    print(json.dumps({
        "metric": "ms per metric pass (dictionary similarity + capacity)", "workload": args.workload, "desc": desc,
        "value": ms, "unit": "ms", "pairs": len(plist), "dictionaries": M, "n": n, "d": d,
        "arith": args.arith, "steps": K, "warmup": W,
        "tflops_algorithmic": flops / (ms * 1e-3) / 1e12,
        "deviation_from_fp64": dev_of(res["mcs_ab"], res["mcs_ba"], cap),
        "stock_torch_gpu": {
            "fp32": {"ms": ms_fp32, "tflops_algorithmic": flops / (ms_fp32 * 1e-3) / 1e12,
                     "deviation_from_fp64": dev_of(*ref32)},
            "tf32": {"ms": ms_tf32, "tflops_algorithmic": flops / (ms_tf32 * 1e-3) / 1e12,
                     "deviation_from_fp64": dev_of(*reftf)},
            "passes_timed": k_ref},
        "speedup_vs_stock_fp32": ms_fp32 / ms, "speedup_vs_stock_tf32": ms_tf32 / ms,
        "gpu": name, "power_limit_w": limit,
    }), flush=True)


EVAL_WORKLOADS = {
    # name: (M, n, d, rows, description)
    "eval_cfg2": (16, 4096, 512, 1 << 20, "16 seeded config-2 TiedSAE dictionaries (4096 x 512) over 2^20 fp16 rows, "
                                          "segment 1000"),
    "eval_cfg5": (1, 32768, 2048, 1 << 18, "one 32768 x 2048 TiedSAE dictionary over 2^18 fp16 rows, segment 1000"),
}


def run_eval(args):
    """Scores of exported dictionaries on a set of activations: the engine's evaluate_dicts pass over all rows and all
    dictionaries, against the reference's per-dictionary op sequence (calc_moments_streaming, then
    fraction_variance_unexplained and mean_nonzero_activations, fp32 torch on the same GPU; the last two over 8192-row
    pieces, since the whole set's dense code would not fit) timed on one dictionary."""
    import sparse_coding_b200 as S
    from oracle import eval_oracle as O
    from sparse_coding_b200 import metrics as MT

    dev, K, W = setup(args)
    M, n, d, N, desc = EVAL_WORKLOADS[args.workload]
    lds = [S.FunctionalTiedSAE.to_learned_dict(p, b) for p, b in make_models(S.FunctionalTiedSAE, M, d, n, seed=0)]
    for ld in lds:
        ld.to_device(dev)
    x = activations(N, d, dev)

    ms, _ = timed(lambda: MT.evaluate_dicts(lds, x, segment=1000, arith=args.arith), K, W)

    def stock(ld, xs):
        """the reference's op sequence for one dictionary (standard_metrics.py:305-314, 482-511)"""
        moments = [torch.zeros(ld.n_feats, device=dev) for _ in range(5)]
        times, mean, m2, m3, m4 = moments
        seen = 0
        for i in range(0, xs.shape[0], 1000):
            c = ld.encode(xs[i:i + 1000].float())
            bm = c.mean(dim=0)
            times += (bm != 0).float()
            mean = (seen * mean + 1000 * bm) / (seen + 1000)
            m2 = (seen * m2 + 1000 * (c ** 2).mean(dim=0)) / (seen + 1000)
            m3 = (seen * m3 + 1000 * (c ** 3).mean(dim=0)) / (seen + 1000)
            m4 = (seen * m4 + 1000 * (c ** 4).mean(dim=0)) / (seen + 1000)
            seen += 1000
        sq = torch.zeros((), dtype=torch.float64, device=dev)
        nz = torch.zeros(ld.n_feats, device=dev)
        for i in range(0, xs.shape[0], 8192):
            b = xs[i:i + 8192].float()
            sq += (b - ld.predict(b)).pow(2).sum().double()
            nz += (ld.encode(ld.center(b)) != 0).float().sum(dim=0)
        xf = xs.float()
        total = (xf - xf.mean(dim=0)).pow(2).sum().double()
        return (sq / total).float(), mean

    k_ref = 1
    tf32 = torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cuda.matmul.allow_tf32 = False
        ms_fp32, _ = timed(lambda: stock(lds[0], x), k_ref, 1)
        torch.backends.cuda.matmul.allow_tf32 = True
        ms_tf32, _ = timed(lambda: stock(lds[0], x), k_ref, 1)
        sub = x[:16384 + 500]                                       # deviation from fp64 on a subsample, dictionary 0
        m64 = {"kind": "tied", "encoder": lds[0].encoder.double(), "encoder_bias": lds[0].encoder_bias.double()}
        f64 = O.fraction_variance_unexplained(m64, sub.double())
        mean64 = O.calc_moments_streaming(m64, sub.double(), 1000)[1]
        dev_of = lambda f, mean: {"fvu_rel": float(abs(float(f) - float(f64)) / float(f64)),
                                  "mean_max_rel": float((mean.double() - mean64).abs().max() / mean64.abs().max())}
        r = MT.evaluate_dicts(lds[:1], sub, segment=1000, arith=args.arith)[0]
        dev_engine = dev_of(r["fvu"], r["mean"])
        dev_tf32 = dev_of(*stock(lds[0], sub))
        torch.backends.cuda.matmul.allow_tf32 = False
        dev_fp32 = dev_of(*stock(lds[0], sub))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    name, limit = card_info(0)
    print(json.dumps({
        "metric": "ms per evaluation pass (evaluate_dicts: FVU, counts, moments of every dictionary)",
        "workload": args.workload, "desc": desc, "value": ms, "unit": "ms", "dictionaries": M, "n": n, "d": d,
        "rows": N, "rows_per_s": N / (ms * 1e-3), "arith": args.arith, "steps": K, "warmup": W,
        "deviation_from_fp64": dev_engine,
        "stock_torch_gpu_per_dictionary": {"fp32": {"ms": ms_fp32, "deviation_from_fp64": dev_fp32},
                                           "tf32": {"ms": ms_tf32, "deviation_from_fp64": dev_tf32},
                                           "passes_timed": k_ref},
        "speedup_vs_stock_fp32": ms_fp32 * M / ms, "speedup_vs_stock_tf32": ms_tf32 * M / ms,
        "gpu": name, "power_limit_w": limit,
    }), flush=True)


INTERP_WORKLOADS = {
    # name: (M, n, d, fragments, description)
    "interp_cfg2": (16, 4096, 512, 50000, "16 seeded config-2 TiedSAE dictionaries (4096 x 512) over 50 000 fragments "
                                          "of 64 fp16 rows, 20 top + 20 random records per feature"),
    "interp_cfg5": (1, 32768, 2048, 50000, "one 32768 x 2048 TiedSAE dictionary over 50 000 fragments of 64 fp16 rows, "
                                           "20 top + 20 random records per feature"),
}


def run_interp(args):
    """Record selection: the engine's top_activating_fragments pass over all fragments and dictionaries, against the
    reference's op sequence on the same GPU for one dictionary, batched over 128 fragments per call (encode, amax over
    the tokens, then topk over the fragments per feature; fp32 and TF32), and the reference's literal loop, one
    fragment per encode with the maxima and per-token values copied to host fp16 tables, on 1 000 fragments."""
    import sparse_coding_b200 as S
    from sparse_coding_b200 import metrics as MT

    dev, K, W = setup(args)
    M, n, d, G, desc = INTERP_WORKLOADS[args.workload]
    L = 64
    lds = [S.FunctionalTiedSAE.to_learned_dict(p, b) for p, b in make_models(S.FunctionalTiedSAE, M, d, n, seed=0)]
    for ld in lds:
        ld.to_device(dev)
    N = G * L
    x = activations(N, d, dev)

    ms, res = timed(lambda: MT.top_activating_fragments(lds, x, arith=args.arith), K, W)
    skipped = float(sum(r["skipped"].float().mean() for r in res) / M)
    del res

    def stock(ld):
        """fragment maxima of one dictionary, 128 fragments per encode, then the top 20 fragments of each feature"""
        fmax = torch.empty(G, n, device=dev)
        for g0 in range(0, G, 128):
            g1 = min(G, g0 + 128)
            c = ld.encode(x[g0 * L:g1 * L].float())
            fmax[g0:g1] = c.reshape(g1 - g0, L, n).amax(1)
        return torch.topk(fmax, 20, dim=0).indices

    def literal(ld, frags=1000):
        """the reference's loop: one fragment per encode, maxima and per-token values to host fp16 tables"""
        maxes = np.zeros((frags, n), dtype=np.float16)
        table = np.zeros((frags, n * L), dtype=np.float16)
        for g in range(frags):
            c = ld.encode(x[g * L:(g + 1) * L].float())
            maxes[g] = torch.max(c, dim=0)[0].cpu().numpy()
            table[g] = c.cpu().numpy().flatten()
        return maxes

    tf32 = torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cuda.matmul.allow_tf32 = False
        ms_fp32, _ = timed(lambda: stock(lds[0]), 1, 1)
        ms_literal, _ = timed(lambda: literal(lds[0]), 1, 0)
        torch.backends.cuda.matmul.allow_tf32 = True
        ms_tf32, _ = timed(lambda: stock(lds[0]), 1, 1)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    name, limit = card_info(0)
    print(json.dumps({
        "metric": "ms per record-selection pass (top_activating_fragments of every dictionary)",
        "workload": args.workload, "desc": desc, "value": ms, "unit": "ms", "dictionaries": M, "n": n, "d": d,
        "fragments": G, "fragment_len": L, "rows": N, "rows_per_s": N / (ms * 1e-3), "arith": args.arith, "steps": K,
        "warmup": W, "skipped_fraction": skipped,
        "stock_torch_gpu_per_dictionary": {"batched_fp32_ms": ms_fp32, "batched_tf32_ms": ms_tf32,
                                           "literal_loop_ms_per_1000_fragments": ms_literal,
                                           "what": "maxima + topk only: no per-token records, no random records"},
        "speedup_vs_batched_fp32": ms_fp32 * M / ms, "speedup_vs_batched_tf32": ms_tf32 * M / ms,
        "speedup_vs_literal_loop": ms_literal * (G / 1000) * M / ms,
        "gpu": name, "power_limit_w": limit,
    }), flush=True)


BASELINE_WORKLOADS = {
    # name: (d, rows or fragments, description)
    "eval_baselines": (512, 1 << 20, "ICAEncoder (fitted by the engine), RandomDict(512) and IdentityReLU(512) over 2^20 "
                                     "fp16 rows in one evaluate_dicts pass, segment 1000"),
    "interp_baselines": (512, 50000, "ICAEncoder, RandomDict(512) and IdentityReLU(512): top_activating_fragments over "
                                     "50 000 fragments of 64 fp16 rows, 20 top + 20 random records per feature"),
}
SKLEARN_ROWS = 1 << 16     # host subsample the reference's ICA encode is timed on, scaled to the workload's rows


def baseline_dicts(d, x, dev):
    """[ICAEncoder fitted by the engine on the first 2^18 rows (at most 50 iterations), RandomDict, IdentityReLU]."""
    import warnings

    import sparse_coding_b200 as S  # noqa: F401  (the engine's library)
    from sparse_coding_b200.ica import ICAEncoder
    from sparse_coding_b200.learned_dict import IdentityReLU, RandomDict
    np.random.seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ica = ICAEncoder(d, device=dev, max_iter=50).fit(x[: 1 << 18])
    torch.manual_seed(0)
    rd, ir = RandomDict(d), IdentityReLU(d)
    rd.to_device(dev)
    ir.to_device(dev)
    return [ica, rd, ir]


def sklearn_ica_encode_ms(x, rows):
    """ms of the reference's ICA encode (ica.py:30-34: the rows to host fp64, StandardScaler.transform,
    FastICA.transform, the code back to the device) over ``rows`` rows, timed on SKLEARN_ROWS rows and scaled; sklearn's
    objects are fitted on a small subsample (their values do not change the cost). None without sklearn."""
    import time
    import warnings
    try:
        from sklearn.decomposition import FastICA
        from sklearn.preprocessing import StandardScaler
    except ImportError:
        return None
    sub = x[:SKLEARN_ROWS]
    scaler = StandardScaler()
    fit = scaler.fit_transform(sub[:8192].float().cpu().numpy().astype(np.float64))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ica = FastICA(max_iter=5).fit(fit)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    c = ica.transform(scaler.transform(sub.float().cpu().numpy().astype(np.float64)))
    torch.tensor(c, device=x.device)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 * rows / sub.shape[0]


def run_baselines(args):
    """The baselines of sweep_baselines.py in one engine pass, against the reference's op sequences on the same GPU:
    RandomDict and IdentityReLU as fp32 / TF32 torch (evaluation: calc_moments_streaming's loop over segments of 1000
    rows, then FVU and mean_nonzero_activations over 8192-row pieces; record selection: 128 fragments per encode, amax
    over the tokens, topk over the fragments), ICA as the reference's sklearn encode on the host, scaled from a
    subsample (its moment and top-k arithmetic, on the GPU, is not added)."""
    from sparse_coding_b200 import metrics as MT

    dev, K, W = setup(args)
    d, size, desc = BASELINE_WORKLOADS[args.workload]
    interp = args.workload.startswith("interp")
    L = 64
    N = size * L if interp else size
    x = activations(N, d, dev)
    lds = baseline_dicts(d, x, dev)
    if interp:
        ms, res = timed(lambda: MT.top_activating_fragments(lds, x, arith=args.arith), K, W)
        del res
    else:
        ms, res = timed(lambda: MT.evaluate_dicts(lds, x, segment=1000, arith=args.arith), K, W)
        del res
    torch_lds = lds[1:]

    def stock_eval(ld):
        D = ld.get_learned_dict().to(dev)
        times, mean, m2, m3, m4 = (torch.zeros(ld.n_feats, device=dev) for _ in range(5))
        seen = 0
        for i in range(0, N, 1000):
            c = ld.encode(x[i:i + 1000].float())
            bm = c.mean(dim=0)
            times += (bm != 0).float()
            mean = (seen * mean + 1000 * bm) / (seen + 1000)
            m2 = (seen * m2 + 1000 * (c ** 2).mean(dim=0)) / (seen + 1000)
            m3 = (seen * m3 + 1000 * (c ** 3).mean(dim=0)) / (seen + 1000)
            m4 = (seen * m4 + 1000 * (c ** 4).mean(dim=0)) / (seen + 1000)
            seen += 1000
        sq = torch.zeros((), dtype=torch.float64, device=dev)
        nz = torch.zeros(ld.n_feats, device=dev)
        for i in range(0, N, 8192):
            b = x[i:i + 8192].float()
            c = ld.encode(b)
            sq += (b - c @ D).pow(2).sum().double()
            nz += (c != 0).float().sum(dim=0)
        return sq, mean

    def stock_interp(ld):
        n = ld.n_feats
        fmax = torch.empty(size, n, device=dev)
        for g0 in range(0, size, 128):
            g1 = min(size, g0 + 128)
            fmax[g0:g1] = ld.encode(x[g0 * L:g1 * L].float()).reshape(g1 - g0, L, n).amax(1)
        return torch.topk(fmax, 20, dim=0).indices

    stock = stock_interp if interp else stock_eval
    tf32 = torch.backends.cuda.matmul.allow_tf32
    ref = {}
    try:
        for name, allow in (("fp32", False), ("tf32", True)):
            torch.backends.cuda.matmul.allow_tf32 = allow
            ref[name] = {type(ld).__name__: timed(lambda: stock(ld), 1, 1)[0] for ld in torch_lds}
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    ica_ms = sklearn_ica_encode_ms(x, N)
    ref_total = {k: sum(v.values()) + (ica_ms or 0.0) for k, v in ref.items()}
    gpu, limit = card_info(0)
    print(json.dumps({
        "metric": "ms per pass over the three baselines (" + ("top_activating_fragments" if interp else "evaluate_dicts")
                  + ")", "workload": args.workload, "desc": desc, "value": ms, "unit": "ms", "d": d, "rows": N,
        "rows_per_s": N / (ms * 1e-3), "arith": args.arith, "steps": K, "warmup": W,
        "reference": {"torch_gpu_ms": ref, "ica_sklearn_host_ms": ica_ms,
                      "ica_sklearn": {"scaled": True, "timed_rows": SKLEARN_ROWS,
                                      "what": "encode only: rows to host fp64, StandardScaler.transform, FastICA.transform, "
                                              "code to the device"} if ica_ms is not None else "sklearn not installed",
                      "total_ms": ref_total},
        "speedup_vs_reference_fp32": ref_total["fp32"] / ms, "speedup_vs_reference_tf32": ref_total["tf32"] / ms,
        "gpu": gpu, "power_limit_w": limit,
    }), flush=True)


TOPFVU_WORKLOADS = {
    # name: (M, n, d, rows, n_top, description)
    "topfvu_cfg2": (16, 4096, 512, 1 << 20, 2, "16 seeded config-2 TiedSAE dictionaries (4096 x 512) over 2^20 fp16 rows, "
                                               "n_top = 2"),
}
TOPFVU_REF_ROWS = 1 << 16     # rows the reference's function is timed on per call (its three [rows, n] fp32 tensors)


def run_topfvu(args):
    """The top- and rest-feature FVU (standard_metrics.py:316-342): evaluate_dicts(n_top) over all rows and dictionaries,
    the same call without n_top (the difference is the cost of the second pass), and the reference's function per
    dictionary in fp32 and TF32 on the same GPU, timed on TOPFVU_REF_ROWS rows and scaled to the workload's rows."""
    import sparse_coding_b200 as S
    from oracle import top_fvu_oracle as TO
    from sparse_coding_b200 import metrics as MT

    dev, K, W = setup(args)
    M, n, d, N, k, desc = TOPFVU_WORKLOADS[args.workload]
    lds = [S.FunctionalTiedSAE.to_learned_dict(p, b) for p, b in make_models(S.FunctionalTiedSAE, M, d, n, seed=0)]
    for ld in lds:
        ld.to_device(dev)
    x = activations(N, d, dev)
    ms_split, r = timed(lambda: MT.evaluate_dicts(lds, x, arith=args.arith, n_top=k), K, W)
    ms_plain, _ = timed(lambda: MT.evaluate_dicts(lds, x, arith=args.arith), K, W)

    def stock(ld, xs):
        """the reference's function, written out (standard_metrics.py:316-342)"""
        c = ld.encode(ld.center(xs))
        idxs = torch.argsort(c.mean(dim=0), descending=True)
        c_top = torch.zeros_like(c)
        c_top[:, idxs[:k]] = c[:, idxs[:k]]
        c_rest = torch.zeros_like(c)
        c_rest[:, idxs[k:]] = c[:, idxs[k:]]
        x_top, x_rest = ld.center(ld.decode(c_top)), ld.center(ld.decode(c_rest))
        var = (xs - xs.mean(dim=0)).pow(2).mean()
        return (xs - x_top).pow(2).mean() / var, (xs - x_rest).pow(2).mean() / var

    sub = x[:TOPFVU_REF_ROWS].float()
    tf32 = torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cuda.matmul.allow_tf32 = False
        ms_fp32, _ = timed(lambda: stock(lds[0], sub), 3, 1)
        torch.backends.cuda.matmul.allow_tf32 = True
        ms_tf32, _ = timed(lambda: stock(lds[0], sub), 3, 1)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    # deviation of the engine from fp64 on a subsample, dictionary 0
    small = x[:16384 + 500]
    m64 = {"kind": "tied", "encoder": lds[0].encoder.double(), "encoder_bias": lds[0].encoder_bias.double()}
    t64, r64, _ = TO.fraction_variance_unexplained_top_activating(m64, small.double(), k)
    e = MT.evaluate_dicts(lds[:1], small, arith=args.arith, n_top=k)[0]
    scale = N / TOPFVU_REF_ROWS
    name, limit = card_info(0)
    print(json.dumps({
        "metric": "ms per evaluation pass with the top- and rest-feature FVU (evaluate_dicts(n_top))",
        "workload": args.workload, "desc": desc, "value": ms_split, "unit": "ms", "dictionaries": M, "n": n, "d": d,
        "rows": N, "n_top": k, "arith": args.arith, "steps": K, "warmup": W,
        "without_n_top_ms": ms_plain, "second_pass_ms": ms_split - ms_plain,
        "fvu_top_rest_dict0": [float(r[0]["fvu_top"]), float(r[0]["fvu_rest"])],
        "deviation_from_fp64": {"fvu_top_rel": abs(float(e["fvu_top"]) / float(t64) - 1),
                                "fvu_rest_rel": abs(float(e["fvu_rest"]) / float(r64) - 1)},
        "stock_torch_gpu_per_dictionary": {"rows_timed": TOPFVU_REF_ROWS, "fp32_ms": ms_fp32 * scale,
                                           "tf32_ms": ms_tf32 * scale, "scaled_by": scale},
        "speedup_vs_stock_fp32": ms_fp32 * scale * M / ms_split, "speedup_vs_stock_tf32": ms_tf32 * scale * M / ms_split,
        "gpu": name, "power_limit_w": limit,
    }), flush=True)


INTERFERENCE_WORKLOADS = {
    # name: (M, n, d, rows, description)
    "interference_cfg2": (16, 4096, 512, 1 << 20, "16 seeded config-2 TiedSAE dictionaries (4096 x 512) over 2^20 fp16 "
                                                  "rows"),
}
SPARSE_FRAC = 50 / 4096
INTERFERENCE_REF_ROWS = (2000, 1 << 14)   # the sample log_standard_metrics takes, and a larger one to scale from


def run_interference(args):
    """The expected interference (big_sweep.py:43-57): evaluate_dicts(interference=True) over all rows and dictionaries,
    the same call without it, and the reference's function per dictionary in fp32 and TF32 on the same GPU (code from
    the dictionary's own encode), on each of INTERFERENCE_REF_ROWS rows; the larger is also scaled to the workload's."""
    import sparse_coding_b200 as S
    from oracle import interference_oracle as IO
    from sparse_coding_b200 import metrics as MT

    dev, K, W = setup(args)
    M, n, d, N, desc = INTERFERENCE_WORKLOADS[args.workload]
    lds = [S.FunctionalTiedSAE.to_learned_dict(p, b) for p, b in make_models(S.FunctionalTiedSAE, M, d, n, seed=0)]
    x = activations(N, d, dev)
    for ld in lds:
        # untrained dictionaries fire on about half the features: set each bias so that its feature fires on SPARSE_FRAC
        # of a sample's rows (L0 about 50, as trained config-2 dictionaries), where the per-row work is what it will be
        ld.to_device(dev)
        pre = x[:8192].float() @ ld.get_learned_dict().T
        ld.encoder_bias = -pre.kthvalue(int(pre.shape[0] * (1.0 - SPARSE_FRAC)), dim=0).values
    print(f"interference_cfg2: dictionaries ready, mean L0 of dictionary 0 on the sample "
          f"{float((lds[0].encode(x[:8192].float()) != 0).sum(1).float().mean()):.1f}", file=sys.stderr, flush=True)
    ms_with, r = timed(lambda: MT.evaluate_dicts(lds, x, arith=args.arith, interference=True), K, W)
    print(f"interference_cfg2: {ms_with:.0f} ms per pass with interference", file=sys.stderr, flush=True)
    ms_plain, _ = timed(lambda: MT.evaluate_dicts(lds, x, arith=args.arith), K, W)

    def stock(dictionary, batch):
        """the reference's function, written out (big_sweep.py:43-57)"""
        norms = torch.norm(dictionary, 2, dim=-1)
        normed_weights = dictionary / torch.clamp(norms, 1e-8)[:, None]
        cosines = torch.einsum("ij,kj->ik", normed_weights, normed_weights)
        totals = torch.einsum("ij,bj->bi", cosines**2, batch)
        capacities = batch / torch.clamp(totals, min=1e-8)
        nonzero_count = batch.count_nonzero(dim=0).float()
        return capacities.sum(dim=0) / torch.clamp(nonzero_count, min=1.0)

    w0 = lds[0].get_learned_dict()
    ref = {}
    tf32 = torch.backends.cuda.matmul.allow_tf32
    try:
        for rows in INTERFERENCE_REF_ROWS:
            c = lds[0].encode(x[:rows].float())
            for mode in ("fp32", "tf32"):
                torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
                ms, _ = timed(lambda: stock(w0, c), 5, 2)
                ref[f"{mode}_ms_{rows}_rows"] = ms
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    big = INTERFERENCE_REF_ROWS[-1]
    scale = N / big
    # deviation of the engine from fp64 on a subsample, dictionary 0 (the drop-in on the same code)
    c = lds[0].encode(x[:big].float())
    want = IO.expected_interference(w0, c)
    got = S.calc_expected_interference(w0, c)
    live = want != 0
    l0 = float((c != 0).sum(1).float().mean())
    name, limit = card_info(0)
    print(json.dumps({
        "metric": "ms per evaluation pass with the expected interference (evaluate_dicts(interference=True))",
        "workload": args.workload, "desc": desc, "value": ms_with, "unit": "ms", "dictionaries": M, "n": n, "d": d,
        "rows": N, "arith": args.arith, "steps": K, "warmup": W, "mean_l0_dict0": l0,
        "without_interference_ms": ms_plain, "interference_ms": ms_with - ms_plain,
        "mean_interference_dict0": float(r[0]["expected_interference"].mean()),
        "dropin_deviation_from_fp64_rel": float(((got.double() - want) / want)[live].abs().max()),
        "stock_torch_gpu_per_dictionary": dict(ref, scaled_fp32_ms=ref[f"fp32_ms_{big}_rows"] * scale,
                                               scaled_tf32_ms=ref[f"tf32_ms_{big}_rows"] * scale, scaled_by=scale),
        "speedup_vs_stock_fp32": ref[f"fp32_ms_{big}_rows"] * scale * M / ms_with,
        "speedup_vs_stock_tf32": ref[f"tf32_ms_{big}_rows"] * scale * M / ms_with,
        "gpu": name, "power_limit_w": limit,
    }), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="mmcs_cfg2",
                    choices=sorted(MMCS_WORKLOADS) + sorted(EVAL_WORKLOADS) + sorted(INTERP_WORKLOADS) +
                    sorted(BASELINE_WORKLOADS) + sorted(TOPFVU_WORKLOADS) + sorted(INTERFERENCE_WORKLOADS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--arith", default="auto", choices=["auto", "bf16x3", "f16f8"])
    args = ap.parse_args()
    if args.workload in INTERFERENCE_WORKLOADS:
        run_interference(args)
    elif args.workload in TOPFVU_WORKLOADS:
        run_topfvu(args)
    elif args.workload in BASELINE_WORKLOADS:
        run_baselines(args)
    elif args.workload in INTERP_WORKLOADS:
        run_interp(args)
    else:
        (run_eval if args.workload in EVAL_WORKLOADS else run_mmcs)(args)


if __name__ == "__main__":
    main()
