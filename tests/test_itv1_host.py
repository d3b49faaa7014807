"""image_transformer_v1 on the CPU: config merge, state-dict layout and signatures against the reference, the oracle against the
reference's recorded outputs (oracle/make_golden_itv1.py), the options the native engine refuses, and the two folds the engine runs v1
through (QKNorm as cosine-sim attention, interleaved RoPE as half-split RoPE on permuted rows), in float64."""
import inspect
import json
import math

import pytest
import torch

import k_diffusion as K
from conftest import GOLDEN, load_npz
from oracle import itv1_oracle as V
from oracle.fixtures import synth_sd

META = json.loads((GOLDEN / "itv1_meta.json").read_text())
CONFIGS = META["configs"]
NAMES = sorted(CONFIGS)


def raw_config(name):
    """the config as a user would write it: what load_config merged, minus the keys it adds"""
    cfg = json.loads(json.dumps(CONFIGS[name]["config"]))
    return {"model": {k: cfg["model"][k] for k in ("type", "input_channels", "input_size", "patch_size", "width", "depth", "sigma_data",
                                                   "sigma_min", "sigma_max")},
            "dataset": {"num_classes": cfg["dataset"]["num_classes"]}}


@pytest.mark.parametrize("name", NAMES)
def test_load_config_merges_like_the_reference(name):
    assert K.config.load_config(raw_config(name)) == CONFIGS[name]["config"]


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_keys_and_shapes_match_the_reference(name):
    model = K.config.make_model(K.config.load_config(raw_config(name)))
    assert isinstance(model, K.models.ImageTransformerDenoiserModelV1)
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == CONFIGS[name]["shapes"]
    assert list(model.state_dict()) == list(CONFIGS[name]["shapes"])


def test_signatures_match_the_reference():
    cls = K.models.ImageTransformerDenoiserModelV1
    assert str(inspect.signature(cls.__init__)) == META["api"]["__init__"]
    assert str(inspect.signature(cls.forward)) == META["api"]["forward"]


def test_constructor_defaults_match_the_reference():
    model = K.models.ImageTransformerDenoiserModelV1(1, 128, 256, 3, 3, [2, 2])
    sd = model.state_dict()
    assert torch.equal(sd["blocks.0.self_attn.qk_norm.scale"], torch.full((2,), math.log(10.0)))
    want = torch.linspace(math.log(math.pi), math.log(5 * math.pi), 16).expand(2, 16)      # axial_rope.py:77-82
    assert torch.equal(sd["blocks.0.self_attn.pos_emb.freqs_h"], want) and torch.equal(sd["blocks.0.self_attn.pos_emb.freqs_w"], want)
    for k in ("out_proj.weight", "blocks.0.self_attn.out_proj.weight", "blocks.0.ff.down_proj.weight", "blocks.0.ff.norm.linear.weight"):
        assert not sd[k].any(), k                                                        # zero-initialised in the reference
    assert model.sigma_data == 1.0 and model.num_classes == 0


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_outputs(name):
    z = load_npz(f"itv1_{name}.npz")
    cfg = CONFIGS[name]["config"]
    sd = synth_sd(CONFIGS[name]["shapes"], 1)
    den = V.make_denoiser(sd, cfg["model"])
    kw = {"class_cond": z["class_cond"]} if "class_cond" in z else {}
    with torch.no_grad():
        torch.testing.assert_close(den(z["x"], z["sigma"], **kw), z["denoised"], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(den(z["x"], z["sigma"], aug_cond=z["aug_cond"], **kw), z["denoised_aug"], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(V.model_forward(sd, cfg["model"], z["x"], z["sigma"], **kw), z["inner"], rtol=1e-5, atol=1e-6)


def test_oracle_heun_matches_reference():
    from oracle import kdiff_oracle as O
    z = load_npz("itv1_mnist.npz")
    cfg = CONFIGS["mnist"]["config"]
    den = V.make_denoiser(synth_sd(CONFIGS["mnist"]["shapes"], 1), cfg["model"])
    with torch.no_grad():
        got = O.sample_heun(den, z["heun_x"], z["heun_sigmas"], dict(class_cond=z["heun_class_cond"]))
    torch.testing.assert_close(got, z["heun"], rtol=1e-4, atol=1e-4)


def test_synth_weights_exercise_the_clamp():
    """some heads of every synthetic config sit above ln 100, where the reference clamps the QKNorm scale"""
    sd = synth_sd(CONFIGS["cifar"]["shapes"], 1)
    s = torch.cat([v for k, v in sd.items() if k.endswith("qk_norm.scale")])
    assert (s > math.log(100.0)).any() and (s < math.log(100.0)).any()


def test_refusals():
    base = raw_config("edge")
    with pytest.raises(ValueError, match="augment_wrapper"):
        K.config.load_config({**base, "model": {**base["model"], "augment_wrapper": True}})
    with pytest.raises(ValueError, match="multiple of"):
        K.config.load_config({**base, "model": {**base["model"], "width": 96}})
    cfg = K.config.load_config(base)
    with pytest.raises(ValueError, match="d_ff"):
        K.config.make_model({**cfg, "model": {**cfg["model"], "d_ff": 0}})
    with pytest.raises(ValueError, match="augment_wrapper"):
        K.config.make_model({**cfg, "model": {**cfg["model"], "augment_wrapper": True}})
    with pytest.raises(ValueError, match="multiple of"):
        K.models.ImageTransformerDenoiserModelV1(1, 96, 256, 3, 3, [2, 2])
    model = K.config.make_model(cfg)
    with pytest.raises(TypeError):
        model(torch.zeros(1, 3, 24, 40), torch.ones(1), mapping_cond=torch.zeros(1, 4))
    with pytest.raises(TypeError, match="mapping_cond"):
        model._check_cond(None, torch.zeros(1, 4))


@pytest.mark.parametrize("clamped", [False, True])
def test_folds_equal_qknorm_and_interleaved_rope(clamped):
    """reference QKNorm + interleaved AxialRoPE + SDPA logits on the original rows == the engine's cosine sim + half-split RoPE of R = 64
    on the permuted rows, in float64, for random q, k, positions, frequencies and scales"""
    g = torch.Generator().manual_seed(5 + clamped)
    nh, T, e = 3, 37, V.D_HEAD
    dt = torch.float64
    q = torch.randn(2, nh, T, e, generator=g, dtype=dt) * 3
    k = torch.randn(2, nh, T, e, generator=g, dtype=dt) * 0.5
    pos = torch.rand(T, 2, generator=g, dtype=dt) * 2 - 1
    fh = torch.randn(nh, e // 4, generator=g, dtype=dt)
    fw = torch.randn(nh, e // 4, generator=g, dtype=dt)
    s = torch.rand(nh, generator=g, dtype=dt) * 3 + (3.5 if clamped else 0.5)
    if clamped:
        assert (s > V.MAX_LOG_SCALE).any()
    theta = V.rope_theta(pos, fh, fw)
    qr, kr = V.apply_rope(V.qk_norm(q, s), theta), V.apply_rope(V.qk_norm(k, s), theta)
    want = qr @ kr.transpose(-1, -2) / math.sqrt(e)                                       # SDPA's logits
    perm = V.head_permutation(e)
    scale, eps = V.fold_qknorm(s, e)
    table = V.fold_rope(fh, fw)
    qe, ke = V.engine_qk(q[..., perm], pos, scale, eps, table), V.engine_qk(k[..., perm], pos, scale, eps, table)
    torch.testing.assert_close(qe @ ke.transpose(-1, -2), want, rtol=1e-10, atol=1e-10)
    # the engine's q, k are the reference's rotated q, k in the permuted column order, up to the 1/sqrt(e) the logit carries
    torch.testing.assert_close(qe, qr[..., perm] * e ** -0.25, rtol=1e-10, atol=1e-12)
    assert (scale <= 100 * (1 + 1e-12)).all()
