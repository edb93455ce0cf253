"""sc_datasets/random_dataset.py of the reference, backed by sparse_coding_b200.synthetic (the classes pickle under
this module's name)."""
from sparse_coding_b200.synthetic import (RandomDatasetGenerator, SparseMixDataset,  # noqa: F401
                                          generate_corr_matrix, generate_correlated_dataset, generate_noise_dataset,
                                          generate_rand_dataset, generate_rand_feats)
