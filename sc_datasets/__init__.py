"""Import shim: the reference's package name. A ``generator.pt`` written by HoagyC/sparse_coding pickles
``sc_datasets.random_dataset.SparseMixDataset``; plotting scripts and sweeps do
``from sc_datasets.random_dataset import SparseMixDataset``. These modules re-export the GPU generators of
``sparse_coding_b200.synthetic`` under those names (see INTEGRATION.md)."""
from sparse_coding_b200.synthetic import RandomDatasetGenerator, SparseMixDataset  # noqa: F401
