"""Boundary proof against the REFERENCE's engine layout (SURVEY.md 8(b); VERDICT r1 item 9).

The reference's `DiffusionEngine.__init__` (sgm/models/video_diffusion.py:35-105), run unmodified on the reduced-width
V3D_512 config below with its own `target:` strings, builds an engine whose `state_dict()` key -> shape map is stored,
as a sha256 digest with its entry counts, in tests/golden/reference_engine_state_dict.json (written by
oracle/make_golden_state_dict.py from the reference checkout).
The drop-in engine built from the drop-in targets of INTEGRATION.md section A is checked against it:

  * the SAME `state_dict()` keys and shapes (network, first-stage decoder, everything else);
  * `load_state_dict(strict=True)` of a checkpoint with the reference's layout, and the weights round-trip;
  * `init_from_ckpt` (the safetensors branch of video_diffusion.py:123-168) loads such a checkpoint with no missing /
    unexpected keys.

CPU only (construction and weight plumbing; no kernels run).
"""
import copy
import hashlib
import json
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

GOLDEN = ROOT / "tests" / "golden" / "reference_engine_state_dict.json"
WIDTH, DEC_CH, T = 64, 64, 4


def _config(prefix: str, first_stage_prefix: str):
    """scripts/pub/configs/V3D_512.yaml:17-146 with the `target:` prefix of the hot-path components as a parameter
    (reduced widths: construction cost only)."""
    dm = prefix + ".modules.diffusionmodules."
    return dict(
        scale_factor=0.18215, disable_first_stage_autocast=True, input_key="latents", log_keys=[], en_and_decode_n_samples_a_time=T,
        denoiser_config={"target": dm + "denoiser.Denoiser",
                         "params": {"scaling_config": {"target": dm + "denoiser_scaling.VScalingWithEDMcNoise"}}},
        network_config={"target": dm + "video_model.VideoUNet",
                        "params": dict(adm_in_channels=768, num_classes="sequential", use_checkpoint=False, in_channels=8,
                                       out_channels=4, model_channels=WIDTH, attention_resolutions=[4, 2, 1],
                                       num_res_blocks=2, channel_mult=[1, 2, 4, 4], num_head_channels=64,
                                       use_linear_in_transformer=True, transformer_depth=1, context_dim=1024,
                                       spatial_transformer_attn_type="softmax", extra_ff_mix_layer=True,
                                       use_spatial_context=True, merge_strategy="learned_with_images",
                                       video_kernel_size=[3, 1, 1])},
        first_stage_config={
            "target": first_stage_prefix + ".models.autoencoder.AutoencodingEngine",
            "params": {
                "loss_config": {"target": "torch.nn.Identity"},
                "regularizer_config": {"target": first_stage_prefix + ".modules.autoencoding.regularizers."
                                                 "DiagonalGaussianRegularizer"},
                "encoder_config": {"target": "torch.nn.Identity"},
                "decoder_config": {"target": prefix + ".modules.autoencoding.temporal_ae.VideoDecoder",
                                   "params": dict(attn_type="vanilla", double_z=True, z_channels=4, resolution=256,
                                                  in_channels=3, out_ch=3, ch=DEC_CH, ch_mult=[1, 2, 4, 4],
                                                  num_res_blocks=2, attn_resolutions=[], dropout=0.0,
                                                  video_kernel_size=[3, 1, 1])}}},
        sampler_config={"target": dm + "sampling.EulerEDMSampler",
                        "params": {"num_steps": 3,
                                   "discretization_config": {"target": dm + "discretizer.EDMDiscretization",
                                                             "params": {"sigma_max": 700.0}},
                                   "guider_config": {"target": dm + "guiders.LinearPredictionGuider",
                                                     "params": {"max_scale": 3.5, "min_scale": 3.5, "num_frames": T}}}},
    )


def layout_digest(layout) -> str:
    """sha256 over the sorted `key:shape` lines of a state-dict layout."""
    lines = "\n".join(f"{k}:{','.join(str(int(d)) for d in shape)}" for k, shape in sorted(layout.items()))
    return hashlib.sha256(lines.encode()).hexdigest()


@pytest.fixture(scope="module")
def golden():
    return json.loads(GOLDEN.read_text())


@pytest.fixture(scope="module")
def drop():
    from v3d_b200.sgm.models.video_diffusion import DiffusionEngine

    torch.manual_seed(0)
    return DiffusionEngine(**copy.deepcopy(_config("v3d_b200.sgm", "v3d_b200.sgm")))


@pytest.fixture(scope="module")
def layout(drop, golden):
    """The drop-in engine's layout, once it is shown to be the reference's."""
    mine = {k: tuple(v.shape) for k, v in drop.state_dict().items()}
    assert len(mine) == golden["entries"] and layout_digest(mine) == golden["sha256"]
    return mine


def _hot_path_items(sd):
    return {k: tuple(v) for k, v in sd.items()
            if k.startswith("model.diffusion_model.") or k.startswith("first_stage_model.decoder.")}


def _reference_shaped_weights(layout):
    """Seeded values in the reference's layout (a stand-in for a checkpoint the reference engine would write)."""
    g = torch.Generator().manual_seed(0)
    return {k: torch.randn(shape, generator=g) if shape else torch.randn((), generator=g) for k, shape in sorted(layout.items())}


def test_reference_loader_builds_dropins_with_identical_state_dict(drop, golden):
    import v3d_b200.decoder
    import v3d_b200.sampling
    import v3d_b200.unet

    # the drop-in targets constructed OUR classes
    assert isinstance(drop.model.diffusion_model, v3d_b200.unet.VideoUNet)
    assert isinstance(drop.first_stage_model.decoder, v3d_b200.decoder.VideoDecoder)
    assert isinstance(drop.sampler, v3d_b200.sampling.EulerEDMSampler)
    assert isinstance(drop.denoiser, v3d_b200.sampling.Denoiser)
    mine = {k: tuple(v.shape) for k, v in drop.state_dict().items()}
    hot = _hot_path_items(mine)
    # the network and the first-stage decoder have the reference's keys and shapes
    assert len(hot) > 1000 and len(hot) == golden["hot_path_entries"]
    assert layout_digest(hot) == golden["hot_path_sha256"]
    # nothing else differs either (conditioner stub has no weights; the denoiser / sampler hold no parameters)
    assert len(mine) == golden["entries"] and layout_digest(mine) == golden["sha256"]


def test_strict_load_state_dict_round_trip(drop, layout):
    sd = {k: v.reshape(layout[k]) for k, v in _reference_shaped_weights(layout).items()}
    missing, unexpected = drop.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    back = drop.state_dict()
    for k in ("model.diffusion_model.input_blocks.0.0.weight", "model.diffusion_model.out.2.bias",
              "first_stage_model.decoder.conv_in.weight", "first_stage_model.decoder.conv_out.time_mix_conv.weight"):
        assert torch.equal(back[k], sd[k]), k


def test_reference_init_from_ckpt_loads_into_dropins(layout, tmp_path):
    from safetensors.torch import save_file

    from v3d_b200.sgm.models.video_diffusion import DiffusionEngine

    want = {k: v.reshape(layout[k]).contiguous() for k, v in _reference_shaped_weights(layout).items()}
    path = str(tmp_path / "v3d_small.safetensors")
    save_file(want, path)
    eng = DiffusionEngine(ckpt_path=path, **copy.deepcopy(_config("v3d_b200.sgm", "v3d_b200.sgm")))
    got = eng.state_dict()
    for k, v in want.items():
        assert torch.equal(got[k], v), k
