from sparse_coding_b200.learned_dict import IdentityReLU, LearnedDict, RandomDict, Rotation, TiedSAE, UntiedSAE  # noqa: F401
