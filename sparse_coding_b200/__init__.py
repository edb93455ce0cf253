"""sparse_coding_b200 — H100-native engine for the ensemble sparse-autoencoder sweep of HoagyC/sparse_coding.

Public names mirror the reference's ``autoencoders`` package for the hot path only (SURVEY.md §8):
DictSignature / FunctionalEnsemble (ensemble.py), FunctionalSAE / FunctionalTiedSAE / FunctionalTiedCenteredSAE /
FunctionalPositiveTiedSAE / masked variants (sae_ensemble.py), TopKEncoder / TopKLearnedDict (topk_encoder.py),
LearnedDict / TiedSAE / UntiedSAE (learned_dict.py), plus the driver loop pieces of big_sweep.py (train_loop.py),
on-device metrics (metrics.py) and the synthetic datasets of sc_datasets/random_dataset.py generated on the GPU
(synthetic.py)."""
from . import metrics
from .metrics import (batched_calc_feature_n_ever_active, calc_expected_interference, calc_moments_streaming,
                      code_correlation, evaluate_dicts,
                      fraction_variance_unexplained, fraction_variance_unexplained_top_activating,
                      mean_nonzero_activations, r_squared, top_activating_fragments)
from .ensemble import CodeProxy, FunctionalEnsemble, optim_str_to_func, stack_dict, unstack_dict
from .learned_dict import LearnedDict, TiedSAE, UntiedSAE
from .optim import AdamConfig, adam
from .sae_ensemble import (FunctionalMaskedSAE, FunctionalMaskedTiedSAE, FunctionalPositiveTiedSAE, FunctionalSAE,
                           FunctionalTiedCenteredSAE, FunctionalTiedSAE)
from .signatures import DictSignature
from .synthetic import (RandomDatasetGenerator, SparseMixDataset, SyntheticChunks, generate_corr_matrix,
                        generate_correlated_dataset, generate_noise_dataset, generate_rand_dataset, generate_rand_feats,
                        generate_synthetic_dataset, init_synthetic_dataset)
from .topk_encoder import TopKEncoder, TopKLearnedDict

__all__ = [
    "AdamConfig", "CodeProxy", "DictSignature", "FunctionalEnsemble", "FunctionalMaskedSAE", "FunctionalMaskedTiedSAE",
    "FunctionalPositiveTiedSAE", "FunctionalSAE", "FunctionalTiedCenteredSAE", "FunctionalTiedSAE", "LearnedDict",
    "TiedSAE", "TopKEncoder", "TopKLearnedDict", "UntiedSAE",
    "adam", "batched_calc_feature_n_ever_active", "calc_expected_interference", "calc_moments_streaming",
    "code_correlation", "evaluate_dicts",
    "fraction_variance_unexplained", "fraction_variance_unexplained_top_activating", "mean_nonzero_activations", "optim_str_to_func", "r_squared", "stack_dict",
    "top_activating_fragments", "unstack_dict",
    "RandomDatasetGenerator", "SparseMixDataset", "SyntheticChunks", "generate_corr_matrix",
    "generate_correlated_dataset", "generate_noise_dataset", "generate_rand_dataset", "generate_rand_feats",
    "generate_synthetic_dataset", "init_synthetic_dataset",
]
