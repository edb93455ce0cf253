from sparse_coding_b200.pca import BatchedPCA, PCAEncoder, calc_pca  # noqa: F401
