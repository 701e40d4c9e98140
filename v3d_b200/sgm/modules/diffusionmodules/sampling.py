from v3d_b200.sampling import EulerEDMSampler, HeunEDMSampler  # noqa: F401  (reference: sampling.py:24-133,214-237)
from v3d_b200.sampling import (  # noqa: F401  (reference: sampling.py:136-211,240-365)
    DPMPP2MSampler,
    DPMPP2SAncestralSampler,
    EulerAncestralSampler,
    LinearMultistepSampler,
)
