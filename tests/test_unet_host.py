"""image_v1 U-Net on the CPU: config merge, state-dict layout and signatures against the reference, the oracle against the
reference's recorded outputs (oracle/make_golden_unet.py), and the options the native engine refuses."""
import inspect
import json

import pytest
import torch

import k_diffusion as K
from conftest import GOLDEN, load_npz
from oracle import kdiff_oracle as O
from oracle import unet_oracle as U
from oracle.fixtures import synth_sd

META = json.loads((GOLDEN / "unet_configs.json").read_text())
NAMES = sorted(META)


@pytest.mark.parametrize("name", NAMES)
def test_load_config_merges_like_the_reference(name):
    assert K.config.load_config(json.loads(json.dumps(META[name]["config"]))) == META[name]["config"]


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_keys_and_shapes_match_the_reference(name):
    model = K.config.make_model(K.config.load_config(META[name]["config"]))
    assert isinstance(model, K.augmentation.KarrasAugmentWrapper)
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == META[name]["shapes"]


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_outputs(name):
    z = load_npz(f"unet_{name}.npz")
    mcfg = META[name]["config"]["model"]
    den = U.make_denoiser(U.strip_prefix(synth_sd(META[name]["shapes"], 1)), mcfg)
    with torch.no_grad():
        O_plain = den(z["x"], z["sigma"])
        O_aug = den(z["x"], z["sigma"], aug_cond=z["aug_cond"])
    torch.testing.assert_close(O_plain, z["denoised"], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(O_aug, z["denoised_aug"], rtol=1e-5, atol=1e-6)
    assert not torch.equal(z["denoised"], z["denoised_aug"])


def test_oracle_heun_trajectory_matches_reference():
    z = load_npz("unet_mnist.npz")
    den = U.make_denoiser(U.strip_prefix(synth_sd(META["mnist"]["shapes"], 1)), META["mnist"]["config"]["model"])
    torch.testing.assert_close(O.sample_heun(den, z["heun_x"], z["heun_sigmas"]), z["heun"], rtol=1e-5, atol=1e-5)


def test_constructor_and_forward_signatures_match_the_reference():
    """reference models/image_v1.py:90,135 and augmentation.py:93,97"""
    sig = lambda f: [(p.name, p.default) for p in inspect.signature(f).parameters.values()]
    e = inspect.Parameter.empty
    assert sig(K.models.ImageDenoiserModelV1.__init__) == [
        ("self", e), ("c_in", e), ("feats_in", e), ("depths", e), ("channels", e), ("self_attn_depths", e), ("cross_attn_depths", None),
        ("mapping_cond_dim", 0), ("unet_cond_dim", 0), ("cross_cond_dim", 0), ("dropout_rate", 0.), ("patch_size", 1), ("skip_stages", 0),
        ("has_variance", False)]
    assert sig(K.models.ImageDenoiserModelV1.forward) == [
        ("self", e), ("input", e), ("sigma", e), ("mapping_cond", None), ("unet_cond", None), ("cross_cond", None), ("cross_cond_padding", None),
        ("return_variance", False)]
    assert sig(K.augmentation.KarrasAugmentWrapper.forward) == [
        ("self", e), ("input", e), ("sigma", e), ("aug_cond", None), ("mapping_cond", None), ("kwargs", e)]


def test_unsupported_options_raise():
    cfg = K.config.load_config(META["mnist"]["config"])
    for key in ("cross_cond_dim", "unet_cond_dim"):
        bad = json.loads(json.dumps(cfg))
        bad["model"][key] = 4
        with pytest.raises(NotImplementedError):
            K.config.make_model(bad)
    model = K.config.make_model(cfg)
    with pytest.raises(ValueError):
        model.set_precision("bf16")
    assert model.set_precision("auto") is model
    assert model.resolved_precision() == K._native.PREC_FP32
    with pytest.raises(NotImplementedError):
        model.inner_model(torch.zeros(1, 1, 28, 28), torch.ones(1), return_variance=True)
    with pytest.raises(NotImplementedError):
        model.denoise_jvp(None, None, None, 1.0)
    with pytest.raises(NotImplementedError):
        model.denoise_vjp(None, None, None, 1.0)
    assert K.Denoiser(model).is_native()


@pytest.mark.parametrize("missing", ["input_channels", "input_size", "mapping_out", "depths", "channels", "self_attn_depths"])
def test_incomplete_image_v1_config_raises_value_error(missing):
    m = dict(META["mnist"]["config"]["model"])
    del m[missing]
    with pytest.raises(ValueError, match=missing):
        K.config.load_config({"model": m})
