"""PixelNeRF scene conditioning without a GPU: the oracle against the reference fixtures, the state_dict layout, and
the host logic of PixelNeRF / PixelNeRFEmbedder / ExtraConditioner through the stand-ins of tests/emu_ops.py
(key order, the `rgb` key, the uc zeros, the "(b t)" repeat, and the jitter draws of the c and uc passes)."""
from __future__ import annotations

import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))

import emu_ops  # noqa: E402
from oracle import ref_pixelnerf as R  # noqa: E402

GOLDEN = Path(__file__).parent / "golden"
TAGS = ["scene_s1", "scene_s3"]


def _fixture(tag):
    return torch.load(GOLDEN / f"{tag}.pt", weights_only=False)


def _embedder(cs, sampler=None):
    from v3d_b200.sgm.modules.encoders.modules import PixelNeRFEmbedder

    emb = PixelNeRFEmbedder(
        {"target": "v3d_b200.sgm.modules.encoders.pixelnerf.ImageEncoder"},
        {"target": "v3d_b200.sgm.modules.encoders.pixelnerf.PixelNeRF",
         "params": dict(num_samples_per_ray=cs["ns"], feature_dim=cs["C"], use_feats_std=cs["use_feats_std"],
                        use_pos_emb=cs["use_pos_emb"])},
        render_size=cs["render_size"], num_video_frames=cs["T"])
    if sampler is not None:
        emb.pixelnerf_encoder.jitter_sampler = sampler
    return emb


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_meets_reference_fixture(tag):
    fx = _fixture(tag)
    cs = fx["case"]
    rgb, fe = R.embedder(fx["state_dict"], fx["inputs"], cs["render_size"], fx["jitter"].reshape(cs["ns"], -1),
                         cs["ns"], use_std=cs["use_feats_std"], use_pe=cs["use_pos_emb"])
    assert float((rgb - fx["rgb"]).abs().max() / fx["rgb"].abs().max()) <= 2e-4
    assert float((fe - fx["feats"]).abs().max() / fx["feats"].abs().max()) <= 2e-4


@pytest.mark.parametrize("tag", TAGS)
def test_state_dict_layout_matches_reference(tag):
    fx = _fixture(tag)
    sd = _embedder(fx["case"]).pixelnerf_encoder.state_dict()
    assert list(sd.keys()) == list(fx["reference_state_dict_shapes"].keys())
    assert {k: tuple(v.shape) for k, v in sd.items()} == fx["reference_state_dict_shapes"]
    for k in ("positional_encoder._freqs", "positional_encoder._phases"):
        assert torch.equal(sd[k], fx["state_dict"][k])


@pytest.mark.parametrize("tag", TAGS)
def test_module_through_standins_meets_fixture(tag):
    fx = _fixture(tag)
    cs = fx["case"]
    shapes = []

    def sampler(shape, dev):
        shapes.append(tuple(shape))
        return fx["jitter"].clone()

    emb = _embedder(cs, sampler)
    emb.pixelnerf_encoder.load_state_dict(fx["state_dict"])
    with emu_ops.patched() as launches:
        n0 = launches.copy()
        rgb, fe = emb(fx["inputs"])
    calls = launches - n0
    assert dict(calls) == {"pixelnerf_rays": 1, "pixelnerf_render": 1, "pixelnerf_decode": 1}
    assert shapes == [(cs["ns"], cs["B"] * cs["T"], cs["render_size"] ** 2, 1)]
    assert rgb.shape == fx["rgb"].shape and fe.shape == fx["feats"].shape
    for name, a, b in (("rgb", rgb, fx["rgb"]), ("feats", fe, fx["feats"])):  # bf16 weights / activations
        whole, varying = R.fixture_errors(a, b)
        assert whole <= R.FIXTURE_REL_L2 and varying <= R.FIXTURE_REL_L2, f"{tag} {name}: {whole:.2e} / {varying:.2e}"


@pytest.mark.parametrize("tag", TAGS)
def test_fixture_bound_rejects_wrong_sources(tag):
    # the fixtures' weights are large enough that the sources decide the output: zeroed or swapped source images
    # miss the bound by a wide margin, so an embedder reading the wrong frame or dropping the gather cannot pass
    fx = _fixture(tag)
    cs = fx["case"]
    for what, inp in R.altered_sources(fx["inputs"]).items():
        rgb, fe = R.embedder(fx["state_dict"], inp, cs["render_size"], fx["jitter"].reshape(cs["ns"], -1),
                             cs["ns"], use_std=cs["use_feats_std"], use_pe=cs["use_pos_emb"])
        for name, a, b in (("rgb", rgb, fx["rgb"]), ("feats", fe, fx["feats"])):
            varying = R.fixture_errors(a, b)[1]
            assert varying > 3 * R.FIXTURE_REL_L2, f"{tag} {what} {name}: {varying:.2e}"


def test_extra_conditioner_meets_reference(tag="scene_s1"):
    # (c, uc) of the real ExtraConditioner around the real PixelNeRFEmbedder (oracle/make_golden_scene.py): key order,
    # the `rgb` key, the "(b t)" repeats, the concatenation order and the uc zeros; the embedder through the stand-ins
    from v3d_b200.sgm.modules import ExtraConditioner

    fx = _fixture(tag)
    cs, ref = fx["case"], fx["conditioner"]
    B, T, rs = cs["B"], cs["T"], cs["render_size"]
    draws = []

    def sampler(shape, dev):
        draws.append(tuple(shape))
        return fx["jitter"].clone()

    cond = ExtraConditioner([
        {"input_key": "cond_frames", "target": "v3d_b200.conditioning.IdentityEncoder"},
        {"input_key": "pixelnerf_input", "target": "v3d_b200.sgm.modules.encoders.modules.PixelNeRFEmbedder",
         "params": {"image_encoder_config": {"target": "v3d_b200.sgm.modules.encoders.pixelnerf.ImageEncoder"},
                    "pixelnerf_encoder_config": {
                        "target": "v3d_b200.sgm.modules.encoders.pixelnerf.PixelNeRF",
                        "params": dict(num_samples_per_ray=cs["ns"], feature_dim=cs["C"], use_feats_std=True,
                                       use_pos_emb=True, jitter_sampler=sampler)},
                    "render_size": rs, "num_video_frames": T}},
        {"input_key": "clip", "target": "v3d_b200.conditioning.IdentityEncoder"},
    ])
    cond.embedders[1].pixelnerf_encoder.load_state_dict(fx["state_dict"])
    batch = dict(ref["batch"], pixelnerf_input=fx["inputs"])
    keys = ["cond_frames", "pixelnerf_input", "clip"]
    with emu_ops.patched() as launches:
        n0 = launches.copy()
        c, uc = cond.get_unconditional_conditioning(batch, force_uc_zero_embeddings=keys)
    calls = launches - n0
    # the embedder runs for c and for uc, and draws its jitter both times, in the reference's shape
    assert calls["pixelnerf_render"] == 2 and draws == [(cs["ns"], B * T, rs * rs, 1)] * 2
    assert list(c.keys()) == ref["c_keys"] == ["concat", "rgb", "crossattn"] and list(uc.keys()) == ref["uc_keys"]
    for d, r in ((c, ref["c"]), (uc, ref["uc"])):
        for k in d:
            assert d[k].shape == r[k].shape, k
        # cond_frames repeated "(b t)" first, then the 128 feature channels; clip repeated "(b t)": exact
        assert torch.equal(d["concat"][:, :4], r["concat"][:, :4]) and torch.equal(d["crossattn"], r["crossattn"])
        assert torch.equal(d["concat"][:, 4:] == 0, r["concat"][:, 4:] == 0)
    # rendered parts through the stand-ins (bf16 weights and activations)
    for name, a, b in (("c rgb", c["rgb"], ref["c"]["rgb"]), ("c feats", c["concat"][:, 4:], ref["c"]["concat"][:, 4:]),
                       ("uc rgb", uc["rgb"], ref["uc"]["rgb"])):
        whole, varying = R.fixture_errors(a, b)
        assert whole <= R.FIXTURE_REL_L2 and varying <= R.FIXTURE_REL_L2, f"{name}: {whole:.2e} / {varying:.2e}"
    # uc: every conditioner input zeroed, but `rgb` is set before the zeroing and survives, as in the reference
    assert not uc["concat"].any() and not uc["crossattn"].any() and ref["uc"]["rgb"].any()


def test_unsupported_options_raise():
    from v3d_b200.pixelnerf import PixelNeRF, PixelNeRFEmbedder

    with pytest.raises(NotImplementedError):
        PixelNeRF(interp="bicubic")
    with pytest.raises(NotImplementedError):
        PixelNeRF(padding="reflection")
    with pytest.raises(NotImplementedError):
        PixelNeRF(num_samples_per_ray=1)
    with pytest.raises(NotImplementedError):
        PixelNeRF(feature_dim=96, use_feats_std=True, use_pos_emb=True)  # 231 > 192 MLP inputs
    with pytest.raises(NotImplementedError):
        PixelNeRFEmbedder({"target": "torch.nn.Identity"},
                          {"target": "v3d_b200.sgm.modules.encoders.pixelnerf.PixelNeRF"}, 8, 4)


def test_abi_declares_pixelnerf_entry_points():
    from v3d_b200 import _lib

    header = (Path(__file__).parent.parent / "include" / "v3d_b200.h").read_text()
    for name in ("v3d_pixelnerf_rays", "v3d_pixelnerf_render", "v3d_pixelnerf_decode"):
        assert name in _lib.SIGNATURES and f"int {name}(" in header
