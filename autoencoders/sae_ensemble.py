from sparse_coding_b200.sae_ensemble import (FunctionalMaskedSAE, FunctionalMaskedTiedSAE, FunctionalSAE,  # noqa: F401
                                             FunctionalTiedCenteredSAE, FunctionalTiedSAE)
