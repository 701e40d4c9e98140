"""Golden state-dict layout of the REAL reference engine (TEST INFRASTRUCTURE; needs the reference checkout).

The reference's `DiffusionEngine.__init__` (sgm/models/video_diffusion.py:35-105) is run, unmodified, on the reduced-width
V3D_512 config of tests/test_reference_loader_cpu.py with its own `target:` strings; the sha256 digest of the
`state_dict()` key -> shape map it builds (and its entry counts) is written to tests/golden/reference_engine_state_dict.json,
which the test compares the drop-in engine's map with.

    python -m oracle.make_golden_state_dict
"""
from __future__ import annotations

import copy
import importlib
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from oracle import reference_shim  # noqa: E402


def main() -> None:
    from test_reference_loader_cpu import _config, layout_digest

    reference_shim.install()
    reference_shim._stub("kornia")
    reference_shim._stub("open_clip")
    mods = sys.modules["sgm.modules"]
    enc = importlib.import_module("sgm.modules.encoders.modules")
    # what sgm/modules/__init__.py:1-6 defines (the package __init__ itself is bypassed by the shim: it pulls CLIP)
    mods.GeneralConditioner = enc.GeneralConditioner
    mods.UNCONDITIONAL_CONFIG = {"target": "sgm.modules.GeneralConditioner", "params": {"emb_models": []}}
    vd = importlib.import_module("sgm.models.video_diffusion")
    torch.manual_seed(0)
    ref = vd.DiffusionEngine(**copy.deepcopy(_config("sgm", "sgm")))
    layout = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    hot = [k for k in layout if k.startswith("model.diffusion_model.") or k.startswith("first_stage_model.decoder.")]
    out = ROOT / "tests" / "golden" / "reference_engine_state_dict.json"
    out.write_text(json.dumps({"entries": len(layout), "hot_path_entries": len(hot), "sha256": layout_digest(layout),
                               "hot_path_sha256": layout_digest({k: layout[k] for k in hot})}, indent=1) + "\n")
    print(f"{out}: {len(layout)} entries")


if __name__ == "__main__":
    main()
