from sparse_coding_b200.learned_dict import LearnedDict, Rotation, TiedSAE, UntiedSAE  # noqa: F401
