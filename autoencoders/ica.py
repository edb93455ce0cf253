from sparse_coding_b200.ica import FittedFastICA, FittedScaler, ICAEncoder  # noqa: F401
