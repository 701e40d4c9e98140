from v3d_b200.conditioning import (ConcatTimestepEmbedderND, GeneralConditioner,  # noqa: F401
                                   IdentityEncoder)  # reference: encoders/modules.py:85-206, 937-953
from v3d_b200.clip import FrozenOpenCLIPImageEmbedder, FrozenOpenCLIPImagePredictionEmbedder  # noqa: F401,E402
from v3d_b200.pixelnerf import ExtraConditioner, PixelNeRFEmbedder  # noqa: F401,E402  (reference: encoders/modules.py:1075-1187)
