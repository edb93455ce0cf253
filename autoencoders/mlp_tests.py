from sparse_coding_b200.sae_ensemble import FunctionalPositiveTiedSAE  # noqa: F401
