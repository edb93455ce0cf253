"""fp64 restatement of the reference's ICA baseline (autoencoders/ica.py:18-58: StandardScaler, then FastICA() with its
defaults: parallel updates, logcosh with alpha = 1, whiten="unit-variance" by SVD, max_iter = 200, tol = 1e-4).
Device-agnostic torch: runs on the CPU against tests/golden/ica.pt and on the GPU at scale.

  standardise   z = (x - m) / s, s the population std with 1 where the column is constant
  whitening     from the population covariance C of x: the eigenpairs (lam, u) of the correlation D^-1 C D^-1 in
                descending order, each u signed by its first entry; K = (u / sqrt(N lam))^T (FastICA's whitening_)
                and Kw = diag(1 / sqrt(lam)) u^T D^-1 (whitened rows X1 = Kw (x - m)^T)
  update        W1 = sym(G X1^T / N - diag(mean_b g') W), G = tanh(alpha W X1), g' = alpha (1 - G^2);
                lim = max_i | |(W1 W^T)_ii| - 1 |
  read-out      W /= sqrt(diag(W W^T) / N) per row (the std of the sources), components = W K, mixing = pinv."""
import numpy as np
import torch


def mixed_sources(d, n, seed):
    """[n, d] fp64 rows: d independent unit-variance sources (even ones Laplace, odd ones sparse: Bernoulli(0.2) times
    a normal), mixed by a seeded matrix with singular values 0.3^(i / (d - 1)), from 1 down to 0.3, around a non-zero
    offset. numpy's legacy
    RandomState, so the same seed gives the same rows everywhere."""
    rs = np.random.RandomState(seed)
    lap = rs.laplace(0.0, 1.0 / np.sqrt(2.0), size=(n, d))
    sparse = (rs.uniform(size=(n, d)) < 0.2) * rs.normal(size=(n, d)) / np.sqrt(0.2)
    src = np.where(np.arange(d) % 2 == 0, lap, sparse)
    q1, _ = np.linalg.qr(rs.normal(size=(d, d)))
    q2, _ = np.linalg.qr(rs.normal(size=(d, d)))
    mix = (q1 * 0.3 ** (np.arange(d) / (d - 1))) @ q2
    offset = 2.0 * rs.normal(size=d)
    return torch.from_numpy(src @ mix.T + offset), torch.from_numpy(mix)


def standardise(x):
    """(mean, var, scale) of the rows of ``x`` [N, d] in fp64, as StandardScaler fits them."""
    x = x.double()
    n = x.shape[0]
    m = x.mean(dim=0)
    var = ((x - m) ** 2).mean(dim=0)
    eps = torch.finfo(torch.float64).eps
    constant = var <= n * eps * var + (n * m * eps) ** 2
    scale = torch.where(constant, torch.ones_like(var), var.sqrt())
    return m, var, scale


def whitening(cov, scale, n):
    """(K, Kw, lam) from the population covariance ``cov`` [d, d] of x, the scaler's ``scale`` and the row count."""
    cov = cov.double()
    corr = cov / torch.outer(scale, scale)
    lam, u = torch.linalg.eigh(0.5 * (corr + corr.T))
    lam, u = lam.flip(0), u.flip(1)
    u = u * torch.sign(u[0])
    K = (u / (n * lam).sqrt()).T
    Kw = (u / lam.sqrt()).T / scale
    return K, Kw, lam


def sym_decorrelation(W):
    s, u = torch.linalg.eigh(W @ W.T)
    s = s.clamp(min=torch.finfo(W.dtype).tiny)
    return (u * s.rsqrt()) @ u.T @ W


def update(W, X1, alpha=1.0):
    """(W1, lim) of one parallel FastICA iteration from W over the whitened rows ``X1`` [d, N]."""
    G = torch.tanh(alpha * (W @ X1))
    gp = (alpha * (1 - G * G)).mean(dim=1)
    W1 = sym_decorrelation(G @ X1.T / X1.shape[1] - gp[:, None] * W)
    lim = ((W1 * W).sum(dim=1).abs() - 1).abs().max()
    return W1, float(lim)


def fit(x, w_init, max_iter=200, tol=1e-4, alpha=1.0):
    """The whole fit from ``w_init`` [d, d]: a dict of the scaler's mean / var / scale, K, W (the unmixing after the
    unit-variance read-out), components, mixing, n_iter, the lim of every iteration and the fp64 sources of ``x``."""
    x = x.double()
    n = x.shape[0]
    m, var, scale = standardise(x)
    xc = x - m
    cov = xc.T @ xc / n
    K, Kw, lam = whitening(cov, scale, n)
    X1 = Kw @ xc.T
    W = sym_decorrelation(w_init.double().to(x.device))
    lims = []
    for _ in range(max_iter):
        W, lim = update(W, X1, alpha)
        lims.append(lim)
        if lim < tol:
            break
    W = W / ((W * W).sum(dim=1, keepdim=True) / n).sqrt()
    comp = W @ K
    return {"mean": m, "var": var, "scale": scale, "K": K, "W": W, "components": comp,
            "mixing": torch.linalg.pinv(comp), "n_iter": len(lims), "lims": lims, "lam": lam,
            "sources": (xc / scale) @ comp.T}
