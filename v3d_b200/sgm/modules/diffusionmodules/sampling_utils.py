from v3d_b200.sampling import (  # noqa: F401  (reference: sampling_utils.py:7-43)
    get_ancestral_step,
    linear_multistep_coeff,
    to_d,
    to_neg_log_sigma,
    to_sigma,
)
