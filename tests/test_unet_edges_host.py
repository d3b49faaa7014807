"""image_v1 U-Net edge configs on the CPU (oracle/make_golden_unet.py EDGES): the merged config, the state-dict layout and the oracle
against the reference's recorded outputs, so the oracle's patch_size, skip_stages, mapping_cond, augment-wrapper-off and has_variance
branches are pinned to the reference before the GPU tests hold the engine to the oracle."""
import json

import pytest
import torch

import k_diffusion as K
from conftest import GOLDEN, load_npz
from oracle import unet_oracle as U
from oracle.fixtures import synth_sd

EDGES = json.loads((GOLDEN / "unet_edges.json").read_text())
NAMES = sorted(EDGES)
# recorded output -> (aug_cond given, mapping_cond given)
VARIANTS = {"denoised": (False, False), "denoised_aug": (True, False), "denoised_mc": (False, True), "denoised_aug_mc": (True, True)}


def variant_kwargs(z, key):
    use_aug, use_mc = VARIANTS[key]
    kw = {"aug_cond": z["aug_cond"]} if use_aug else {}
    if use_mc:
        kw["mapping_cond"] = z["mapping_cond"]
    return kw


def test_edges_reach_every_option():
    ms = [EDGES[n]["config"]["model"] for n in NAMES]
    assert {m["patch_size"] for m in ms} == {1, 2} and {m["skip_stages"] for m in ms} == {0, 1}
    assert {m["has_variance"] for m in ms} == {False, True} and {m["augment_wrapper"] for m in ms} == {False, True}
    assert any(m["mapping_cond_dim"] > 0 and m["augment_wrapper"] for m in ms) and any(m["mapping_cond_dim"] > 0 and not m["augment_wrapper"] for m in ms)
    assert any(m["input_size"][0] != m["input_size"][1] for m in ms)


@pytest.mark.parametrize("name", NAMES)
def test_edge_load_config_merges_like_the_reference(name):
    assert K.config.load_config(json.loads(json.dumps(EDGES[name]["config"]))) == EDGES[name]["config"]


@pytest.mark.parametrize("name", NAMES)
def test_edge_state_dict_keys_and_shapes_match_the_reference(name):
    cfg = EDGES[name]["config"]
    model = K.config.make_model(K.config.load_config(cfg))
    assert isinstance(model, K.augmentation.KarrasAugmentWrapper) == cfg["model"]["augment_wrapper"]
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == EDGES[name]["shapes"]


@pytest.mark.parametrize("name", NAMES)
def test_edge_oracle_matches_reference_outputs(name):
    z = load_npz(f"unet_edge_{name}.npz")
    den = U.make_denoiser(U.strip_prefix(synth_sd(EDGES[name]["shapes"], 1)), EDGES[name]["config"]["model"])
    keys = [k for k in VARIANTS if k in z]
    assert len(keys) == 2, keys
    for key in keys:
        with torch.no_grad():
            got = den(z["x"], z["sigma"], **variant_kwargs(z, key))
        torch.testing.assert_close(got, z[key], rtol=1e-5, atol=1e-6, msg=lambda m: f"{name} {key}: {m}")
    assert not torch.equal(z[keys[0]], z[keys[1]])


@pytest.mark.parametrize("channels, attn", [([196], [True]), ([64, 196], [False, True]), ([196, 64], [False, True])])
def test_create_refuses_attention_widths_not_divisible_by_the_head_count(channels, attn):
    """max(1, C // 64) heads must divide the width C (the reference asserts it, layers.py:184): 196 would get 3 heads of 65.  A level
    with self-attention attends at its own width and, in its UBlock's last layer, at the width of the level above."""
    spec = dict(c_in=3, feats_in=32, depths=[1] * len(channels), channels=channels, self_attn_depths=attn, mapping_cond_dim=9, augment=True,
                patch_size=1, skip_stages=0, has_variance=False)
    with pytest.raises(ValueError, match="not divisible by its 3 heads"):
        K._native.UNetEngine(spec)
    K._native.UNetEngine(dict(spec, channels=[192 if c == 196 else c for c in channels]))      # 3 heads of 64
