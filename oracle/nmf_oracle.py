"""fp64 restatement of sklearn's NMF() as the reference's NMFEncoder runs it (coordinate descent, Frobenius loss,
NNDSVDA start, no regularisation, coordinates in order), for the tests and the fixture's checks. TEST INFRASTRUCTURE.

  nndsvda(X)            the start (W0, H0), from the exact SVD (numpy) instead of randomized_svd, which at k = d
                        spans the whole column space and agrees up to rounding
  sweep(W, G, L)        one coordinate-descent sweep over the rows of W with G = H H^T, L = X H^T; returns the
                        violation (sum of |projected gradient|)
  fit(X)                the full fit: (W, H, n_iter, violations, reconstruction error)
  transform(X, H)       the W-update alone from W = 0: (W, n_iter)
  nmf_rows(...)         the fixture's datasets, regenerated from their seeds"""
import numpy as np
import torch


def nndsvda(X, eps=1e-6):
    X = torch.as_tensor(X, dtype=torch.float64)
    U, S, Vh = torch.linalg.svd(X, full_matrices=False)
    k = X.shape[1]
    W = torch.zeros(X.shape[0], k, dtype=torch.float64)
    H = torch.zeros(k, X.shape[1], dtype=torch.float64)
    W[:, 0] = S[0].sqrt() * U[:, 0].abs()
    H[0] = S[0].sqrt() * Vh[0].abs()
    for j in range(1, k):
        x, y = U[:, j], Vh[j]
        xp, yp, xn, yn = x.clamp(min=0), y.clamp(min=0), (-x).clamp(min=0), (-y).clamp(min=0)
        mp, mn = xp.norm() * yp.norm(), xn.norm() * yn.norm()
        if mp > mn:
            u, v, sigma = xp / xp.norm(), yp / yp.norm(), mp
        else:
            u, v, sigma = xn / xn.norm(), yn / yn.norm(), mn
        lbd = (S[j] * sigma).sqrt()
        W[:, j], H[j] = lbd * u, lbd * v
    avg = X.mean()
    W[W < eps] = 0
    H[H < eps] = 0
    W[W == 0] = avg
    H[H == 0] = avg
    return W, H


def sweep(W, G, L):
    """One sweep in place over all rows at once (rows are independent; the violation is summed per coordinate)."""
    viol = 0.0
    for t in range(W.shape[1]):
        grad = W @ G[t] - L[:, t]
        wt = W[:, t]
        pg = torch.where(wt == 0, grad.clamp(max=0), grad)
        viol += float(pg.abs().sum())
        if G[t, t] != 0:
            W[:, t] = (wt - grad / G[t, t]).clamp(min=0)
    return viol


def fit(X, max_iter=200, tol=1e-4, W=None, H=None):
    X = torch.as_tensor(X, dtype=torch.float64)
    if W is None:
        W, H = nndsvda(X)
    W, Ht = W.clone(), H.T.contiguous().clone()
    violations = []
    n_iter = 0
    for n_iter in range(1, max_iter + 1):
        v = sweep(W, Ht.T @ Ht, X @ Ht)
        v += sweep(Ht, W.T @ W, X.T @ W)
        violations.append(v)
        if violations[0] == 0 or v / violations[0] <= tol:
            break
    H = Ht.T.contiguous()
    return {"W": W, "H": H, "n_iter": n_iter, "violations": violations, "err": float((X - W @ H).norm())}


def transform(X, H, max_iter=200, tol=1e-4):
    X = torch.as_tensor(X, dtype=torch.float64)
    H = torch.as_tensor(H, dtype=torch.float64)
    W = torch.zeros(X.shape[0], H.shape[0], dtype=torch.float64)
    G, L = H @ H.T, X @ H.T
    v0, n_iter = None, 0
    for n_iter in range(1, max_iter + 1):
        v = sweep(W, G, L)
        if n_iter == 1:
            v0 = v
        if v0 == 0 or v / v0 <= tol:
            break
    return W, n_iter


def nmf_rows(d, n, seed, rank=None, signed=False, separated=False):
    """fp16 [n, d]: a non-negative mixture of `rank` (default d) non-negative sparse sources with non-negative noise,
    scaled to max ~4. signed: shifted by -1 and rounded to multiples of 1/64, so that x - min(x) is exact in fp16.
    rank < d: columns rank .. d-1 are zero, so d - rank singular values are exactly 0. separated: a nearly diagonal
    mixture with little noise (singular values within a factor of ~6), on which sklearn's fit converges in ~15
    iterations instead of running to its cap."""
    g = torch.Generator().manual_seed(seed)
    r = d if rank is None else rank
    src = torch.rand(n, r, generator=g, dtype=torch.float64) ** 3 * (torch.rand(n, r, generator=g) < 0.4)
    if separated:
        mix = torch.eye(r, dtype=torch.float64) * torch.linspace(2.0, 0.5, r, dtype=torch.float64) + \
            0.05 * torch.rand(r, r, generator=g, dtype=torch.float64) * (torch.rand(r, r, generator=g) < 0.2)
        x = src @ mix + 0.005 * torch.rand(n, r, generator=g, dtype=torch.float64)
    else:
        mix = torch.rand(r, r, generator=g, dtype=torch.float64) * (torch.rand(r, r, generator=g) < 0.5) + \
            torch.eye(r, dtype=torch.float64) * torch.linspace(2.0, 0.5, r, dtype=torch.float64)
        x = src @ mix + 0.02 * torch.rand(n, r, generator=g, dtype=torch.float64)
    x = 4 * x / x.max()
    if signed:
        x = torch.round((x - 1.0) * 64) / 64
    out = torch.zeros(n, d, dtype=torch.float64)
    out[:, :r] = x
    return out.half()
