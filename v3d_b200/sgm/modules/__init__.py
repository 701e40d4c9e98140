

from v3d_b200.pixelnerf import ExtraConditioner  # noqa: E402,F401  (reference: sgm/modules/__init__.py:1)
