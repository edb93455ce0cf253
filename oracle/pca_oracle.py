"""fp64 restatement of BatchedPCA (autoencoders/pca.py:41-110) as the shifted sums the engine accumulates: with a fixed
shift s and v = x - s over N rows, S1 = sum v, S2 = sum v v^T, mean = s + S1 / N and cov = (S2 - S1 S1^T / N) / N (the
population covariance, which the reference's batch merge equals in exact arithmetic). Device-agnostic: runs on the CPU
against tests/golden/pca.pt and on the GPU at scale."""
import torch


def moments(x, shift=None):
    """(mean [d], cov [d, d]) in fp64 of the rows of ``x`` [N, d]; ``shift`` defaults to the column mean of the first
    min(N, 500) rows (any shift gives the same result up to rounding)."""
    x = x.double()
    s = x[:500].mean(dim=0) if shift is None else shift.double()
    v = x - s
    n = x.shape[0]
    s1 = v.sum(dim=0)
    s2 = v.T @ v
    return s + s1 / n, (s2 - torch.outer(s1, s1) / n) / n


def pca(cov):
    """(eigenvalues ascending, eigenvectors in columns) of the symmetrised covariance, fp64."""
    return torch.linalg.eigh((cov + cov.T) / 2)


def get_dict(cov):
    """Rows: the eigenvectors by eigenvalue, descending (BatchedPCA.get_dict)."""
    vals, vecs = pca(cov)
    return vecs[:, torch.argsort(vals, descending=True)].T
