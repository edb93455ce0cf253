from sparse_coding_b200.nmf import FittedNMF, NMFEncoder  # noqa: F401
