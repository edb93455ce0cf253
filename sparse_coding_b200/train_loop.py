"""The sweep's hot loop and its two neighbours: activation-chunk feeding and dictionary export.

Reference behaviour being reproduced (HoagyC/sparse_coding @ 69c5ae0):
  ensemble_train_loop           big_sweep.py:159-199   seeds, one step per sampler batch, optional wandb scalars
  unstacked_to_learned_dicts    big_sweep.py:202-225   export [(LearnedDict, hyperparams)] per model
  make_hyperparam_name          big_sweep.py:75-83     wandb key format
  chunk loop / checkpoints      big_sweep.py:349-384, basic_l1_sweep.py:85-115

What is GPU-native here: the reference gathers every batch on the CPU (``dataset[batch_idxs]``, a 16 MiB fancy-index
copy per step at config 2) and ships it through a pageable, synchronous H2D copy (its ``pin_memory()`` call discards
the result, SURVEY.md Q5). Here the whole chunk (2 GiB as fp16) is made resident in HBM once — staged through pinned
memory on a side stream while the previous chunk is still training — and each batch is a device-side row gather
(libsce ``sce_gather_rows``: fp16->fp32 conversion and optional mean-centring fused) followed by ``step_batch``.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Iterable, List, Optional

import numpy as np
import torch

from . import _lib
from .tracing import nvtx_range


# ----------------------------------------------------------------------------------------------------------------
# naming (wandb keys) — big_sweep.py:75-83
# ----------------------------------------------------------------------------------------------------------------
def format_hyperparam_val(val) -> str:
    return f"{val:.2E}".replace("+", "") if isinstance(val, float) else str(val)


def make_hyperparam_name(setting: dict) -> str:
    return "_".join(f"{k}_{format_hyperparam_val(v)}" for k, v in setting.items())


# ----------------------------------------------------------------------------------------------------------------
# device-side batch gather
# ----------------------------------------------------------------------------------------------------------------
def gather_rows(chunk: torch.Tensor, idx: Optional[torch.Tensor], sub: Optional[torch.Tensor] = None,
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[r] = float32(chunk[idx[r]]) - sub, on the GPU (chunk: CUDA fp16/fp32 [N,d]; idx: CUDA int64 [B])."""
    if not chunk.is_cuda:
        raise RuntimeError("gather_rows runs in the CUDA engine; the chunk must be resident on the GPU")
    if chunk.dtype not in (torch.float16, torch.float32) or not chunk.is_contiguous():
        raise TypeError("chunk must be a contiguous fp16 or fp32 tensor")
    N, d = chunk.shape
    B = N if idx is None else idx.numel()
    if out is None:
        out = torch.empty(B, d, dtype=torch.float32, device=chunk.device)
    if idx is not None:
        idx = idx.to(device=chunk.device, dtype=torch.int64).contiguous()
    if sub is not None:
        sub = sub.to(device=chunk.device, dtype=torch.float32).contiguous()
    stream = C.c_void_p(torch.cuda.current_stream(chunk.device).cuda_stream)
    with torch.cuda.device(chunk.device):
        _lib.check(_lib.load().sce_gather_rows(chunk.data_ptr(), int(chunk.dtype == torch.float16), N, d,
                                               idx.data_ptr() if idx is not None else None, B,
                                               sub.data_ptr() if sub is not None else None, out.data_ptr(), stream),
                   "sce_gather_rows")
    return out


def _to_device_staged(t: torch.Tensor, device, piece_bytes: int = 64 << 20) -> torch.Tensor:
    """Host tensor -> device through two pinned staging buffers (asynchronous copies that overlap the host memcpy
    into the other buffer). A pageable 2 GiB chunk handed to ``tensor.to(device)`` is copied synchronously through
    the driver's small bounce buffers; the reference does exactly that every batch (its ``pin_memory()`` call
    discards the result, SURVEY.md Q5)."""
    if t.is_cuda:
        return t
    if t.is_pinned() or t.numel() * t.element_size() <= piece_bytes:
        return t.to(device, non_blocking=True)
    t = t.contiguous()
    out = torch.empty(t.shape, dtype=t.dtype, device=device)
    flat_src, flat_dst = t.view(-1), out.view(-1)
    piece = max(1, piece_bytes // t.element_size())
    stage = [torch.empty(piece, dtype=t.dtype).pin_memory() for _ in range(2)]
    done = [None, None]
    stream = torch.cuda.current_stream(out.device)
    for k, lo in enumerate(range(0, flat_src.numel(), piece)):
        hi = min(lo + piece, flat_src.numel())
        slot = k & 1
        if done[slot] is not None:
            done[slot].synchronize()
        stage[slot][:hi - lo].copy_(flat_src[lo:hi])
        flat_dst[lo:hi].copy_(stage[slot][:hi - lo], non_blocking=True)
        done[slot] = torch.cuda.Event()
        done[slot].record(stream)
    for ev in done:
        if ev is not None:
            ev.synchronize()          # the staging buffers are freed on return
    return out


_PERM_CACHE: dict = {}      # (rows, seed, device) -> permutation on the device; see _batch_index_lists


def _batch_index_lists(sampler, device=None, perm_cache: Optional[dict] = None) -> Iterable[torch.Tensor]:
    """Index tensors per batch (on ``device`` when given). ``perm_cache``: the reference re-seeds the global RNG at
    the start of every chunk (big_sweep.py:161), so equal-length chunks draw the SAME sampler seed and hence the same
    permutation (SURVEY.md Q7); keyed by (rows, that seed, device) the 2M-element randperm and its upload are done once
    instead of once per chunk — the numbers are identical either way. For the reference's ``BatchSampler(RandomSampler(range(N)), B, drop_last=False)``
    (cluster_runs.py:28-32) the permutation is drawn in one go — the same numbers the reference would see, because
    RandomSampler itself draws one ``torch.randperm`` per epoch — instead of building B-element Python lists."""
    inner = getattr(sampler, "sampler", None)
    bs = getattr(sampler, "batch_size", None)
    if isinstance(sampler, torch.utils.data.BatchSampler) and isinstance(inner, torch.utils.data.RandomSampler) \
            and not inner.replacement and inner.num_samples == len(inner.data_source):
        # what RandomSampler.__iter__ does, minus the 2M-element Python list: seed a private generator from the
        # global RNG (or use the sampler's own), draw one permutation
        n = len(inner.data_source)
        if inner.generator is None:
            seed = int(torch.empty((), dtype=torch.int64).random_().item())
            key = (n, seed, str(device))
            gen = torch.Generator()
            gen.manual_seed(seed)
        else:
            gen, key = inner.generator, None
        perm = perm_cache.get(key) if (perm_cache is not None and key is not None) else None
        if perm is None:
            perm = torch.randperm(n, generator=gen)
            if device is not None:
                perm = perm.to(device, non_blocking=False)  # one upload per chunk; the batches are views of it
            if perm_cache is not None and key is not None:
                if len(perm_cache) >= 4:
                    perm_cache.clear()
                perm_cache[key] = perm
        n_full = n // bs * bs
        for i in range(0, n_full, bs):
            yield perm[i:i + bs]
        if n_full < n and not sampler.drop_last:
            yield perm[n_full:]
        return
    for idxs in sampler:
        t = torch.as_tensor(idxs, dtype=torch.int64)
        yield t if device is None else t.to(device, non_blocking=True)


def ensemble_train_loop(ensemble, cfg, args, ensemble_name, sampler, dataset, progress_counter):
    """Drop-in for big_sweep.py:159-199. ``dataset`` is the chunk ([N,d], CPU or CUDA, fp16/fp32)."""
    torch.set_grad_enabled(False)
    torch.manual_seed(0)       # the reference re-seeds at every call: equal-length chunks get equal shuffles (Q7)
    np.random.seed(0)
    device = torch.device(args["device"])
    use_wandb = bool(getattr(cfg, "use_wandb", False))
    run = cfg.wandb_instance if use_wandb else None
    chunk = dataset if dataset.is_cuda else _to_device_staged(dataset, device)
    if not chunk.is_contiguous():
        chunk = chunk.contiguous()
    for i, batch_idxs in enumerate(_batch_index_lists(sampler, device, _PERM_CACHE)):
        batch = gather_rows(chunk, batch_idxs)
        losses, aux_buffer = ensemble.step_batch(batch)
        if use_wandb:
            num_nonzero = aux_buffer["c"].count_nonzero(dim=-1).float().mean(dim=-1)
            host = {k: v.cpu() for k, v in losses.items()}            # one D2H per key, not one per model
            nnz_host = num_nonzero.cpu()
            log = {}
            for m in range(ensemble.n_models):
                hyperparam_values = {}
                for ep in cfg.ensemble_hyperparams:
                    if ep not in args:
                        raise ValueError(f"Hyperparameter {ep} not found in args")
                    hyperparam_values[ep] = args[ep]
                for bp in cfg.buffer_hyperparams:
                    if bp not in ensemble.buffers:
                        raise ValueError(f"Hyperparameter {bp} not found in buffers")
                    hyperparam_values[bp] = ensemble.buffers[bp][m].item()
                name = make_hyperparam_name(hyperparam_values)
                for k in host:
                    log[f"{ensemble_name}_{name}_{k}"] = host[k][m].item()
                log[f"{ensemble_name}_{name}_num_nonzero"] = nnz_host[m].item()
            run.log(log, commit=True)
        progress_counter.value = i
    check_input_range(ensemble)


def check_input_range(ensemble) -> None:
    """Once per chunk (one small D2H copy): read the device-side health flag — a batch beyond the fp16 range or a
    non-finite loss makes the engine SKIP the affected updates; ``check_health`` then moves an ``arith="auto"``
    ensemble to bf16x3 (warning) or raises for an explicitly chosen arithmetic — and warn when the activations fed to
    an f16f8 plan come close to the limits of its fp16 operand plane (very small magnitudes only cost precision,
    silently)."""
    if hasattr(ensemble, "check_health"):
        ensemble.check_health()
    amax = ensemble.input_absmax() if hasattr(ensemble, "input_absmax") else 0.0
    if hasattr(ensemble, "resolved_arith") and ensemble.resolved_arith() != "f16f8":
        return
    if amax != amax or amax > 3.0e4 or 0.0 < amax < 1.0e-3:
        import warnings
        warnings.warn(f"largest |activation| fed to the f16f8 arithmetic so far is {amax:g}: outside [1e-3, 3e4]; "
                      "construct the FunctionalEnsemble with arith='bf16x3' (fp32 range) for this data", RuntimeWarning)


def unstacked_to_learned_dicts(ensemble, args, ensemble_hyperparams, buffer_hyperparams):
    """big_sweep.py:202-225: one (LearnedDict, {hyperparam: value}) per model, tensors on the CPU."""
    learned_dicts = []
    for params, buffers in ensemble.unstack(device="cpu"):
        hyperparam_values = {}
        for ep in ensemble_hyperparams:
            if ep not in args:
                raise ValueError(f"Hyperparameter {ep} not found in args")
            hyperparam_values[ep] = args[ep]
        for bp in buffer_hyperparams:
            if bp not in buffers:
                raise ValueError(f"Hyperparameter {bp} not found in buffers")
            hyperparam_values[bp] = buffers[bp].item()
        learned_dicts.append((ensemble.sig.to_learned_dict(params, buffers), hyperparam_values))
    return learned_dicts


# ----------------------------------------------------------------------------------------------------------------
# activation-chunk streaming: {folder}/{i}.pt  (fp16 [N,d], activation_dataset.py:499-503)
# ----------------------------------------------------------------------------------------------------------------
def _single_record_offset(path: str, nbytes: int) -> Optional[int]:
    """Byte offset of the one tensor-data record of a torch.save()d file (zip container, records stored uncompressed),
    or None when the file is anything else (several storages, legacy format, compressed)."""
    import zipfile
    try:
        with zipfile.ZipFile(path) as z:
            recs = [i for i in z.infolist() if "/data/" in "/" + i.filename and not i.filename.endswith("/")
                    and i.filename.rsplit("/", 1)[-1].isdigit()]
            if len(recs) != 1 or recs[0].compress_type != zipfile.ZIP_STORED or recs[0].file_size != nbytes:
                return None
            info = recs[0]
        with open(path, "rb") as f:
            f.seek(info.header_offset)
            hdr = f.read(30)
            if hdr[:4] != b"PK\x03\x04":
                return None
            return info.header_offset + 30 + int.from_bytes(hdr[26:28], "little") + int.from_bytes(hdr[28:30], "little")
    except (OSError, zipfile.BadZipFile, ValueError):
        return None


class ChunkStreamer:
    """Iterates over device-resident chunks. While the caller trains on chunk i, a background thread moves chunk i+1
    from disk into one of two HBM buffers (ping-pong; the copy waits for the compute that last read that HBM buffer):
    the file is memory-mapped (``torch.load(mmap=True)``) and streamed in 64 MiB pieces through a small ring of pinned
    staging buffers filled by a few reader threads — the host copies of the next pieces overlap the asynchronous H2D of
    piece p on a side stream, one pass over the bytes on the host, 384 MiB of pinned memory instead of two chunk-sized
    buffers. The training stream only
    waits on the copy-complete event, so disk, host memcpy and H2D all overlap with the GPU work of the previous chunk.

    ``feed="broadcast"`` (torch.distributed initialised, one process per GPU, every rank streaming the SAME chunk
    order — the sweep's situation, cluster_runs.py:100-130): only rank ``src`` reads the file and crosses PCIe; the
    chunk then reaches the other GPUs with one NCCL broadcast over NVLink / NVSwitch on the side stream, issued from
    the staging thread on a process group of its own. ``feed="per_rank"`` (default): every rank reads and copies for
    itself (independent PCIe links, no collective)."""

    PIECE_BYTES = 64 << 20
    RING = 6          # pinned pieces (384 MiB)
    READERS = 4       # threads moving file bytes into them (a single thread copies ~1.5 GB/s out of the page cache)

    def __init__(self, folder: str, order: Iterable[int], device, keep_dtype: bool = True, feed: str = "per_rank",
                 src: int = 0):
        from concurrent.futures import ThreadPoolExecutor
        self.folder, self.order, self.device = folder, list(order), torch.device(device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.keep_dtype = keep_dtype
        if feed not in ("per_rank", "broadcast"):
            raise ValueError("feed must be 'per_rank' or 'broadcast'")
        self.feed, self.src, self._group = "per_rank", src, None
        if feed == "broadcast":
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                self.feed = "broadcast"
                self._group = dist.new_group()          # collective: every rank constructs its streamer
                self._rank = dist.get_rank()
        self.copy_stream = torch.cuda.Stream(self.device)
        self._pool = ThreadPoolExecutor(max_workers=1)
        self._readers = ThreadPoolExecutor(max_workers=self.READERS)
        self._ring, self._ring_ev = [], []   # pinned staging pieces (uint8) and the event of their last H2D
        self._dev = [None, None]
        self._copied = [None, None]     # event: H2D into slot finished (pinned buffer reusable, data visible)
        self._released = [None, None]   # event on the training stream: work reading slot has been enqueued
        self.stage_seconds = []         # host time of every staging call (disk + pinned copy + enqueue), for reports

    def _load(self, chunk_idx: int):
        """(tensor, path, byte offset of its data in the file or None). The tensor is memory-mapped (shape / dtype are
        known, bytes are not read yet); when the file is a plain torch.save of ONE contiguous tensor — the reference's
        chunk format — the offset of its (uncompressed) data record lets the staging loop read() the bytes straight
        into pinned memory: with eight ranks faulting in the same mapped file, page-by-page, the mmap route fed each
        rank at 1.1 GB/s (8 GPUs: 66 % of the device-resident rate), read() has no page faults to take."""
        path = os.path.join(self.folder, f"{chunk_idx}.pt")
        try:
            t = torch.load(path, map_location="cpu", mmap=True)
        except (RuntimeError, TypeError, ValueError):            # legacy (non-zip) serialisation cannot be mapped
            t = torch.load(path, map_location="cpu")
        offset = None
        if self.keep_dtype and t.dtype in (torch.float16, torch.float32) and t.is_contiguous() and t.storage_offset() == 0:
            offset = _single_record_offset(path, t.numel() * t.element_size())
        if not self.keep_dtype or t.dtype not in (torch.float16, torch.float32):
            t = t.float()
        return t.contiguous(), path, offset

    def _stage(self, slot: int, chunk_idx: int):
        with nvtx_range(f"sce.stage_chunk {chunk_idx}"):
            return self._stage_impl(slot, chunk_idx)

    def _stage_impl(self, slot: int, chunk_idx: int):
        import time
        t0 = time.perf_counter()
        torch.cuda.set_device(self.device)
        t, path, offset = self._load(chunk_idx)                   # mapped: shape / dtype known, bytes not read yet
        reader = self.feed == "per_rank" or self._rank == self.src
        if self._dev[slot] is None or self._dev[slot].shape != t.shape or self._dev[slot].dtype != t.dtype:
            self._dev[slot] = torch.empty(t.shape, dtype=t.dtype, device=self.device)
        with torch.cuda.stream(self.copy_stream):
            if self._released[slot] is not None:
                self.copy_stream.wait_event(self._released[slot])
            if reader:
                src = t.view(-1).view(torch.uint8)                # (mapped) bytes of the chunk
                dst = self._dev[slot].view(-1).view(torch.uint8)
                piece = self.PIECE_BYTES
                if not self._ring:
                    self._ring = [torch.empty(piece, dtype=torch.uint8).pin_memory() for _ in range(self.RING)]
                    self._ring_ev = [None] * self.RING

                def fill(k, lo, hi):                              # reader thread: piece k of the file -> pinned piece
                    r = k % self.RING
                    if self._ring_ev[r] is not None:
                        self._ring_ev[r].synchronize()            # the H2D that last read this pinned piece has finished
                    if offset is not None:                        # read(): no page faults (see _load)
                        view = memoryview(self._ring[r].numpy())[:hi - lo]
                        with open(path, "rb", buffering=0) as fh:
                            fh.seek(offset + lo)
                            got = 0
                            while got < hi - lo:
                                n_read = fh.readinto(view[got:])
                                if not n_read:
                                    raise IOError(f"short read in {path}")
                                got += n_read
                    else:
                        self._ring[r][:hi - lo].copy_(src[lo:hi])  # mapped page cache -> pinned (host memcpy)
                    return r

                spans = [(lo, min(lo + piece, src.numel())) for lo in range(0, src.numel(), piece)]
                futs = {}
                ahead = self.RING - 1                             # pieces being read while one is being copied
                for k in range(min(ahead, len(spans))):
                    futs[k] = self._readers.submit(fill, k, *spans[k])
                for k, (lo, hi) in enumerate(spans):
                    r = futs.pop(k).result()
                    dst[lo:hi].copy_(self._ring[r][:hi - lo], non_blocking=True)
                    self._ring_ev[r] = torch.cuda.Event()
                    self._ring_ev[r].record(self.copy_stream)
                    if k + ahead < len(spans):
                        futs[k + ahead] = self._readers.submit(fill, k + ahead, *spans[k + ahead])
            if self.feed == "broadcast":
                import torch.distributed as dist
                dist.broadcast(self._dev[slot], src=self.src, group=self._group)   # enqueued on copy_stream
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        self._copied[slot] = ev
        self.stage_seconds.append(time.perf_counter() - t0)
        return ev

    def __iter__(self):
        if not self.order:
            return
        fut = self._pool.submit(self._stage, 0, self.order[0])
        for i, chunk_idx in enumerate(self.order):
            slot = i & 1
            ev = fut.result()
            if i + 1 < len(self.order):
                fut = self._pool.submit(self._stage, slot ^ 1, self.order[i + 1])   # prefetch in the background
            torch.cuda.current_stream(self.device).wait_event(ev)
            yield chunk_idx, self._dev[slot]
            rel = torch.cuda.Event()
            rel.record(torch.cuda.current_stream(self.device))
            self._released[slot] = rel


class HostBatchPrefetcher:
    """Feeds host-resident batches (pinned fp32 / fp16 [B, d] tensors, e.g. what a DataLoader with ``pin_memory``
    yields) to ``step_batch``: the copy of batch i+1 runs on a side stream while the engine works on batch i, through
    a small ring of device buffers. Yields device tensors valid until the next iteration."""

    def __init__(self, batches: Iterable[torch.Tensor], device, depth: int = 2):
        self.batches, self.device, self.depth = batches, torch.device(device), max(2, int(depth))
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.copy_stream = torch.cuda.Stream(self.device)

    def __iter__(self):
        it = iter(self.batches)
        main = torch.cuda.current_stream(self.device)
        bufs, ready, free = [None] * self.depth, [None] * self.depth, [None] * self.depth
        queue = []

        def issue(slot):
            try:
                h = next(it)
            except StopIteration:
                return False
            if bufs[slot] is None or bufs[slot].shape != h.shape or bufs[slot].dtype != h.dtype:
                bufs[slot] = torch.empty(h.shape, dtype=h.dtype, device=self.device)
            with torch.cuda.stream(self.copy_stream):
                if free[slot] is not None:
                    self.copy_stream.wait_event(free[slot])
                bufs[slot].copy_(h, non_blocking=True)
                ready[slot] = torch.cuda.Event()
                ready[slot].record(self.copy_stream)
            queue.append(slot)
            return True

        nxt = 0
        for _ in range(self.depth - 1):
            if not issue(nxt % self.depth):
                break
            nxt += 1
        while queue:
            if issue(nxt % self.depth):
                nxt += 1
            slot = queue.pop(0)
            main.wait_event(ready[slot])
            yield bufs[slot]
            free[slot] = torch.cuda.Event()
            free[slot].record(main)


class _Counter:
    value = 0


def train_on_chunks(ensemble, args: dict, dataset_folder: str, output_folder: str, batch_size: int,
                    ensemble_hyperparams: List[str], buffer_hyperparams: List[str], n_repetitions: int = 1,
                    center_activations: bool = False, cfg=None, chunk_order: Optional[List[int]] = None,
                    save_schedule: str = "sweep", feed: str = "per_rank", on_chunk_end=None):
    """The chunk loop of ``sweep`` (big_sweep.py:349-384) / ``basic_l1_sweep`` (basic_l1_sweep.py:85-115) for ONE
    ensemble on ONE GPU, with streamed chunks. Writes ``_{i}/learned_dicts.pt`` (+ ``config.yaml`` when ``cfg`` is
    given) on the reference's schedule: last chunk, or chunk count in {8, 16, …, 512}. ``feed``: see
    :class:`ChunkStreamer`; ``on_chunk_end(i, chunk_idx, ensemble)`` runs after the last step of every chunk."""
    import yaml

    device = torch.device(args["device"])
    n_chunks = len([f for f in os.listdir(dataset_folder) if f.endswith(".pt") and f[:-3].isdigit()])
    if chunk_order is None:
        chunk_order = list(np.random.permutation(n_chunks))
        if n_repetitions is not None:
            chunk_order = list(np.tile(chunk_order, n_repetitions))
    os.makedirs(output_folder, exist_ok=True)
    means = None
    cfg = cfg if cfg is not None else type("Cfg", (), {"use_wandb": False})()
    learned_dicts = []
    perm_cache: dict = {}
    for i, (chunk_idx, chunk) in enumerate(ChunkStreamer(dataset_folder, chunk_order, device, feed=feed)):
        if center_activations:
            if means is None:
                means = chunk.float().mean(dim=0)
                torch.save(means.cpu(), os.path.join(output_folder, "means.pt"))
        N = chunk.shape[0]
        sampler = torch.utils.data.BatchSampler(torch.utils.data.RandomSampler(range(N)), batch_size=batch_size,
                                                drop_last=False)
        torch.set_grad_enabled(False)
        torch.manual_seed(0)
        np.random.seed(0)
        with nvtx_range(f"sce.chunk {chunk_idx}"):
            for j, idx in enumerate(_batch_index_lists(sampler, device, perm_cache)):
                batch = gather_rows(chunk, idx, sub=means)
                ensemble.step_batch(batch)
        check_input_range(ensemble)
        if on_chunk_end is not None:
            on_chunk_end(i, chunk_idx, ensemble)      # e.g. the end-of-chunk metric gather (sharding.gather_metrics)
        last = i == len(chunk_order) - 1
        if last or (save_schedule == "sweep" and (i + 1) in [2 ** j for j in range(3, 10)]) or save_schedule == "every":
            # export (a full D2H of the parameters, which also drains the GPU) only when a checkpoint is due
            with nvtx_range("sce.export_learned_dicts"):
                learned_dicts = unstacked_to_learned_dicts(ensemble, args, ensemble_hyperparams, buffer_hyperparams)
            it_folder = os.path.join(output_folder, f"_{i}")
            os.makedirs(it_folder, exist_ok=True)
            torch.save(learned_dicts, os.path.join(it_folder, "learned_dicts.pt"))
            if hasattr(cfg, "__dict__") or isinstance(cfg, dict):
                try:
                    with open(os.path.join(it_folder, "config.yaml"), "w") as f:
                        yaml.dump({k: v for k, v in dict(vars(cfg) if not isinstance(cfg, dict) else cfg).items()
                                   if isinstance(v, (int, float, str, bool, list, type(None)))}, f)
                except Exception:
                    pass
    return learned_dicts


# ----------------------------------------------------------------------------------------------------------------
# resume (the reference can only save dictionaries; Adam state is lost between runs — SURVEY.md §5)
# ----------------------------------------------------------------------------------------------------------------
def save_resume_state(ensemble, path: str) -> None:
    sd = ensemble.state_dict()
    cpu = lambda tree: {k: (cpu(v) if isinstance(v, dict) else v.detach().cpu()) for k, v in tree.items()}
    blob = {"params": cpu(sd["params"]), "buffers": cpu(sd["buffers"]), "optim_states": cpu(sd["optim_states"])}
    # every other key of state_dict() — the reference's (sig, optimizer_kwargs, n_models, no_stacking) and all
    # engine-only settings (adam_count_mode, passes, arith and a bf16x3 fall-back taken earlier, health interval,
    # materialize_code, steps) — so that a resumed run computes exactly as the saved one did
    blob.update({k: v for k, v in sd.items() if k not in ("params", "buffers", "optim_states", "device", "optimizer_func")})
    torch.save(blob, path)


def load_resume_state(path: str, device):
    from .ensemble import FunctionalEnsemble
    from .optim import adam
    blob = torch.load(path, map_location="cpu", weights_only=False)
    dev = lambda tree: {k: (dev(v) if isinstance(v, dict) else v.to(device)) for k, v in tree.items()}
    sd = dict(blob)
    sd.update(device=device, params=dev(blob["params"]), buffers=dev(blob["buffers"]),
              optim_states=dev(blob["optim_states"]), optimizer_func=adam)
    return FunctionalEnsemble.from_state(sd)
