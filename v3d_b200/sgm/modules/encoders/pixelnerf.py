from v3d_b200.pixelnerf import ImageEncoder, PixelNeRF, PositionalEncoding  # noqa: F401  (reference: encoders/pixelnerf.py)
