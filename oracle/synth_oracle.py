"""Restatement of libsce sce_synth_rows (include/sce.h) in numpy, for tests: Philox4x32-10 vectorised over counters,
and from it, for given probabilities, each row's active components and fp32 coefficients (bitwise what the kernel
must produce) and x in fp64 (which the kernel's fp32 FMAs approximate)."""
import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
TAG_THRESH, TAG_VALUE, TAG_STRENGTH, TAG_ZERO, TAG_NOISE, TAG_GAUSS = range(6)
_U32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Four uint32 arrays (broadcast) of Philox4x32-10 of counter (c0, c1, c2, c3) under key (k0, k1)."""
    c = [np.asarray(x, dtype=np.uint64) & _U32 for x in np.broadcast_arrays(c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0) & _U32, np.uint64(k1) & _U32
    for _ in range(10):
        p0 = np.uint64(M0) * c[0]            # < 2**64: exact in uint64
        p1 = np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _U32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _U32]
        k0, k1 = (k0 + np.uint64(W0)) & _U32, (k1 + np.uint64(W1)) & _U32
    return [x.astype(np.uint32) for x in c]


def uniform(x):
    """fp32 (x >> 8) 2^-24: exact."""
    return ((np.asarray(x, dtype=np.uint32) >> 8).astype(np.float64) * 2.0 ** -24).astype(np.float32)


def _keys(seed):
    return seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF


def _draw(seed, rows, comps, tag):
    """uint32 word of component j for each (row, j) of rows [R] x comps [J], counter (j / 4, row lo, row hi, tag)."""
    rows = np.asarray(rows, dtype=np.int64)[:, None]
    comps = np.asarray(comps, dtype=np.int64)[None, :]
    w = philox4x32_10(comps >> 2, rows & 0xFFFFFFFF, rows >> 32, tag, *_keys(seed))
    return np.choose(comps & 3, w)


def box_muller_pairs(w, dtype=np.float64):
    """Standard normals of the columns 4q .. 4q + 3 from the four words of counter q: pairs (0, 1) and (2, 3)."""
    out = []
    for a, b in ((w[0], w[1]), (w[2], w[3])):
        u1 = ((a >> 8).astype(np.float64) + 1.0) * 2.0 ** -24
        u2 = (b >> 8).astype(np.float64) * 2.0 ** -24
        r = np.sqrt(-2.0 * np.log(u1))
        out += [r * np.cos(2 * np.pi * u2), r * np.sin(2 * np.pi * u2)]
    return np.stack(out, axis=-1).astype(dtype)


def noise(seed, rows, d):
    """[R, d] fp64 N(0, 1) of the kernel's noise stream."""
    rows = np.asarray(rows, dtype=np.int64)[:, None]
    q = np.arange(d // 4, dtype=np.int64)[None, :]
    w = philox4x32_10(q, rows & 0xFFFFFFFF, rows >> 32, TAG_NOISE, *_keys(seed))
    return box_muller_pairs(w).reshape(len(rows), d)


def group_gaussians(seed, groups, n):
    """[G, n] fp64 normals of the per-group stream (tag 5, group in the row words)."""
    g = np.asarray(groups, dtype=np.int64)[:, None]
    q = np.arange((n + 3) // 4, dtype=np.int64)[None, :]
    w = philox4x32_10(q, g & 0xFFFFFFFF, g >> 32, TAG_GAUSS, *_keys(seed))
    return box_muller_pairs(w).reshape(len(g), -1)[:, :n]


def synth_rows(feats, probs, group_rows, row0, B, seed, zero_row_rule, noise_scale):
    """(lists, x): lists[i] = (int32 indices ascending, fp32 coefficients) of local row i; x [B, d] fp64.
    feats fp32 [n_gt, d]; probs fp32 [G, n_gt]."""
    feats = np.asarray(feats, dtype=np.float32)
    probs = np.asarray(probs, dtype=np.float32)
    n_gt, d = feats.shape
    rows = row0 + np.arange(B, dtype=np.int64)
    comps = np.arange(n_gt)
    p = probs[np.arange(B) // group_rows]
    active = uniform(_draw(seed, rows, comps, TAG_THRESH)) <= p
    coef = uniform(_draw(seed, rows, comps, TAG_VALUE)) * uniform(_draw(seed, rows, comps, TAG_STRENGTH))  # fp32
    lists = []
    code = np.zeros((B, n_gt), dtype=np.float64)
    k0, k1 = _keys(seed)
    for i in range(B):
        idx = np.nonzero(active[i])[0]
        c = coef[i, idx]
        if idx.size == 0 and zero_row_rule:
            z = philox4x32_10(0, rows[i] & 0xFFFFFFFF, rows[i] >> 32, TAG_ZERO, k0, k1)[0]
            j = int((int(z) * n_gt) >> 32)
            s = uniform(_draw(seed, rows[i:i + 1], [j], TAG_STRENGTH))[0, 0]
            idx, c = np.array([j]), np.array([np.float32(1.0) * s], dtype=np.float32)
        lists.append((idx.astype(np.int32), c.astype(np.float32)))
        code[i, idx] = c
    x = code @ feats.astype(np.float64)
    if noise_scale:
        x = x + np.float64(np.float32(noise_scale)) * noise(seed, rows, d)
    return lists, x
