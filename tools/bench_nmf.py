"""Time NMFEncoder's passes on one resident 2^21-row fp16 chunk (the reference's chunk), per fit iteration and per encode.

    python tools/bench_nmf.py [--d 512 2048] [--rows 2097152] [--repeats 3] [--sk-rows 2048]

Per width, after a warm-up iteration, each timed repeat runs one fit iteration's passes exactly as NMFEncoder.fit does
(per 65536-row block: sce_nmf_project with M = H, the fp32 sce_nmf_cd_sweep of that block of W, sce_nmf_grams; then the
fp64 sweep of H^T), with CUDA events around each phase summed over the blocks, and one encode of an 8192-row batch
(200 sweeps: tol = 0). W starts from the NNDSVDA-like state of a short fit (max_iter = 1), so the sweep sees the sparsity
of a real fit. sklearn's iteration is timed on the host, --repeats times from the same state, on a --sk-rows
subsample: the W-update (_update_coordinate_descent: X H^T, H H^T and the Cython sweep, all linear in the rows) and
the H-update's products X^T W and W^T W are scaled by N / sk_rows, the H-update's sweep over d rows is taken as it is.
The sweeps are single-threaded Cython; the products use numpy's BLAS threads (cpu_cores is reported). One JSON line per
width, with the card's name, power limit and SM clock read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from sparse_coding_b200 import _lib  # noqa: E402
from sparse_coding_b200.nmf import NMFEncoder, _gram  # noqa: E402
from sparse_coding_b200._rowpass import call_rows  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        q = f"nvidia-smi failed: {e}"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--d", type=int, nargs="+", default=[512, 2048])
    ap.add_argument("--rows", type=int, default=1 << 21)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--sk-rows", type=int, default=2048)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    for d in a.d:
        N = a.rows
        g = torch.Generator(device=dev).manual_seed(d)
        src = torch.rand(N, 128, generator=g, device=dev) ** 4
        mix = torch.rand(128, d, generator=g, device=dev) * (torch.rand(128, d, generator=g, device=dev) < 0.1)
        x = (src @ mix + 0.05 * torch.rand(N, d, generator=g, device=dev)).half()
        del src
        enc = NMFEncoder(d, max_iter=1)
        W = enc.fit_transform(x)
        H = torch.as_tensor(enc.nmf.components_, device=dev)
        step = call_rows(d)
        cuts = [(s, min(s + step, N)) for s in range(0, N, step)]
        ws, ws_ptr = _lib.workspace(max(lib.sce_nmf_project_workspace_bytes(d, d, step),
                                        lib.sce_nmf_grams_workspace_bytes(d, d, step)), dev, "ws")
        wsb = ws.numel() - 1024
        cd, cd_ptr = _lib.workspace(lib.sce_nmf_cd_sweep_workspace_bytes(d, step), dev, "cd")
        cdb = cd.numel() - 1024
        st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        shift = torch.zeros(d, dtype=torch.float32, device=dev)
        L = torch.empty(step, d, dtype=torch.float32, device=dev)
        wtw, wtv = (torch.zeros(d, d, dtype=torch.float64, device=dev) for _ in range(2))
        viol = torch.zeros(2, dtype=torch.float64, device=dev)
        ev = lambda: torch.cuda.Event(enable_timing=True)   # noqa: E731

        def iteration(Hc):
            t = {"project": 0.0, "w_sweep": 0.0, "grams": 0.0, "h_sweep": 0.0}
            Hf, G = Hc.float().contiguous(), _gram(Hc).float().contiguous()
            for s, e in cuts:
                e0, e1, e2, e3 = ev(), ev(), ev(), ev()
                e0.record()
                _lib.check(lib.sce_nmf_project(x[s:e].data_ptr(), 1, e - s, d, shift.data_ptr(), Hf.data_ptr(), d, 0,
                                               L.data_ptr(), None, None, ws_ptr, wsb, st), "project")
                e1.record()
                _lib.check(lib.sce_nmf_cd_sweep(W[s:e].data_ptr(), 0, e - s, d, G.data_ptr(), L.data_ptr(), 1,
                                                C.c_double(0.0), viol.data_ptr(), None, cd_ptr, cdb, st), "sweep")
                e2.record()
                _lib.check(lib.sce_nmf_grams(x[s:e].data_ptr(), 1, e - s, d, shift.data_ptr(), W[s:e].data_ptr(), d, 0,
                                             wtw.data_ptr(), wtv.data_ptr(), None, ws_ptr, wsb, st), "grams")
                e3.record()
                torch.cuda.synchronize()
                t["project"] += e0.elapsed_time(e1)
                t["w_sweep"] += e1.elapsed_time(e2)
                t["grams"] += e2.elapsed_time(e3)
            Ht, Lh, wtw_s = Hc.T.contiguous(), wtv.T.contiguous(), (0.5 * (wtw + wtw.T)).contiguous()
            e0, e1 = ev(), ev()
            e0.record()
            _lib.check(lib.sce_nmf_cd_sweep(Ht.data_ptr(), 1, d, d, wtw_s.data_ptr(), Lh.data_ptr(), 1, C.c_double(0.0),
                                            viol.data_ptr(), None, cd_ptr, cdb, st), "h sweep")
            e1.record()
            torch.cuda.synchronize()
            t["h_sweep"] = e0.elapsed_time(e1)
            return t, Ht.T.contiguous()

        _, H = iteration(H)   # warm-up
        iters = []
        for _ in range(a.repeats):
            t, H = iteration(H)
            iters.append(t)
        # encode: 8192 rows, 200 sweeps
        enc.nmf.components_ = H.cpu().numpy()
        enc.nmf.tol, enc.nmf.max_iter = 0.0, 200
        enc._cache = None
        xb = x[:8192]
        enc.transform(xb)
        enc_ms = []
        for _ in range(a.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, n_it = enc.transform(xb)
            enc_ms.append((time.perf_counter() - t0) * 1e3)
        # sklearn's iteration on the host, from a subsample: the W-update (its products and sweep scale with the
        # rows) scaled by N / sk_rows; of the H-update, the products X^T W and W^T W scaled, its d-row sweep as it is
        sk = None
        try:
            import numpy as np
            from sklearn.decomposition._cdnmf_fast import _update_cdnmf_fast
            from sklearn.decomposition._nmf import _update_coordinate_descent
            Xs = x[:a.sk_rows].double().cpu().numpy()
            W0s = W[:a.sk_rows].double().cpu().numpy()
            Ht0 = np.ascontiguousarray(H.T.cpu().numpy())
            scale = N / a.sk_rows
            sk = []
            for _ in range(a.repeats):
                Ws, Hts = W0s.copy(), Ht0.copy()
                t0 = time.perf_counter()
                _update_coordinate_descent(Xs, Ws, Hts, 0.0, 0.0, False, None)
                t1 = time.perf_counter()
                WtW, XtW = Ws.T @ Ws, Xs.T @ Ws
                t2 = time.perf_counter()
                _update_cdnmf_fast(Hts, WtW, XtW, np.arange(d, dtype=np.intp))
                t3 = time.perf_counter()
                sk.append((t1 - t0) * scale + (t2 - t1) * scale + (t3 - t2))
        except ImportError:
            pass
        rng = lambda k: [round(min(i[k] for i in iters), 2), round(max(i[k] for i in iters), 2)]   # noqa: E731
        tot = [sum(i.values()) for i in iters]
        print(json.dumps({"d": d, "rows": N, "card": card(), "cpu_cores": os.cpu_count(),
                          "iteration_ms": [round(min(tot), 1), round(max(tot), 1)],
                          "project_ms": rng("project"), "w_sweep_ms": rng("w_sweep"), "grams_ms": rng("grams"),
                          "h_sweep_ms": rng("h_sweep"), "encode_8192x200_ms": [round(min(enc_ms), 1), round(max(enc_ms), 1)],
                          "encode_sweeps": n_it,
                          "sklearn_iteration_s_scaled": None if sk is None else [round(min(sk), 1), round(max(sk), 1)],
                          "w_nonzero_fraction": round(float((W != 0).float().mean()), 3)}), flush=True)
        del x, W, enc


if __name__ == "__main__":
    main()
