"""The tf32 precision on the CPU: how set_precision, KDB200_PRECISION and the augment wrapper select it for the image_v1 U-Net, that
auto still means fp32, that the transformer refuses it, the tf32 restatement the GPU tests hold the engine to, and that the oracle with
that restatement reproduces the reference's tf32 deviation recorded in tests/golden/tf32_budget.json."""
import json

import pytest
import torch

import k_diffusion as K
from conftest import GOLDEN
from oracle import kdiff_oracle as O
from oracle import unet_oracle as U
from oracle.fixtures import synth_sd
from oracle.make_golden_tf32 import tf32_round, tf32_trunc
from test_unet_edges_host import VARIANTS, variant_kwargs

META = json.loads((GOLDEN / "unet_configs.json").read_text())
EDGES = json.loads((GOLDEN / "unet_edges.json").read_text())
BUDGET = json.loads((GOLDEN / "tf32_budget.json").read_text())
N = K._native


def unet():
    return K.config.make_model(K.config.load_config(META["mnist"]["config"]))


def transformer():
    meta = json.loads((GOLDEN / "cfg1_mnist_shapes.json").read_text())
    inner = K.config.make_model(K.config.load_config(meta["config"]))
    inner.load_state_dict(synth_sd(meta["shapes"], 1))
    return inner


def test_set_precision_selects_tf32_through_the_augment_wrapper(monkeypatch):
    monkeypatch.delenv("KDB200_PRECISION", raising=False)
    model = unet()
    assert isinstance(model, K.augmentation.KarrasAugmentWrapper)
    assert N.PREC_TF32 == 2
    assert model.set_precision("tf32") is model
    assert model.resolved_precision() == model.inner_model.resolved_precision() == N.PREC_TF32
    assert model.inner_model.set_precision("fp32").resolved_precision() == N.PREC_FP32
    assert model.resolved_precision() == N.PREC_FP32
    for auto in (None, "auto"):
        assert model.set_precision(auto).resolved_precision() == N.PREC_FP32
    with pytest.raises(ValueError):
        model.set_precision("bf16")
    with pytest.raises(ValueError):
        model.set_precision("tf16")


def test_environment_selects_tf32_unless_the_model_says_otherwise(monkeypatch):
    model = unet()
    monkeypatch.setenv("KDB200_PRECISION", "tf32")
    assert model.resolved_precision() == N.PREC_TF32
    assert model.set_precision("fp32").resolved_precision() == N.PREC_FP32
    monkeypatch.setenv("KDB200_PRECISION", "auto")
    assert model.set_precision(None).resolved_precision() == N.PREC_FP32
    assert K.models.flags.resolve_precision("tf32", torch.float32) == "tf32"
    assert K.models.flags.resolve_precision(None, torch.float32) == "fp32"


def test_transformer_refuses_tf32(monkeypatch):
    monkeypatch.delenv("KDB200_PRECISION", raising=False)
    inner = transformer()
    with pytest.raises(ValueError, match="tf32"):
        inner.set_precision("tf32").resolved_precision()
    inner.set_precision(None)
    assert inner.resolved_precision() == N.PREC_FP32
    monkeypatch.setenv("KDB200_PRECISION", "tf32")
    with pytest.raises(ValueError, match="tf32"):
        inner.resolved_precision()


def test_tf32_restatement():
    """the restatement of the engine's operand rounding (oracle/make_golden_tf32.py): truncation of activations, round-half-away of weights"""
    ulp = 2.0 ** -10
    x = torch.tensor([1 + ulp / 2, 1 + ulp / 2 + 2.0 ** -20, 1 + 1.5 * ulp, -(1 + ulp / 2), 1 + ulp * 0.49, 3.0], dtype=torch.float64)
    assert tf32_trunc(x).tolist() == [1.0, 1.0, 1 + ulp, -1.0, 1.0, 3.0]
    assert tf32_round(x).tolist() == [1 + ulp, 1 + ulp, 1 + 2 * ulp, -(1 + ulp), 1.0, 3.0]


def reproduced(monkeypatch, sd, mcfg):
    """the oracle's denoiser (fp32) with every Conv2d and the attention at tf32, as oracle/make_golden_tf32.py runs the reference"""
    from test_gpu_unet_tf32 import Tf32Functional
    monkeypatch.setattr(U, "F", Tf32Functional([]))
    return U.make_denoiser(sd, mcfg)


def close_to_budget(got, key):
    """the oracle and the reference differ by fp32 noise, which moves a few operands across a tf32 boundary: 10% of the deviation"""
    assert abs(got - BUDGET[key]) <= 0.1 * BUDGET[key], f"{key}: oracle {got:.4e} vs recorded {BUDGET[key]:.4e}"


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("name", sorted(META))
def test_oracle_reproduces_the_recorded_tf32_budget(name, monkeypatch):
    from conftest import load_npz
    z = load_npz(f"unet_{name}.npz")
    den = reproduced(monkeypatch, U.strip_prefix(synth_sd(META[name]["shapes"], 1)), META[name]["config"]["model"])
    with torch.no_grad():
        close_to_budget(rel_l2(den(z["x"], z["sigma"]), z["denoised"]), f"{name}.denoised")
        close_to_budget(rel_l2(den(z["x"], z["sigma"], aug_cond=z["aug_cond"]), z["denoised_aug"]), f"{name}.denoised_aug")
        if name == "mnist":
            close_to_budget(rel_l2(O.sample_heun(den, z["heun_x"], z["heun_sigmas"]), z["heun"]), "mnist.heun10")


@pytest.mark.parametrize("name", sorted(EDGES))
def test_oracle_reproduces_the_recorded_tf32_budget_of_the_edge_configs(name, monkeypatch):
    from conftest import load_npz
    z = load_npz(f"unet_edge_{name}.npz")
    den = reproduced(monkeypatch, U.strip_prefix(synth_sd(EDGES[name]["shapes"], 1)), EDGES[name]["config"]["model"])
    with torch.no_grad():
        for key in (k for k in VARIANTS if k in z):
            close_to_budget(rel_l2(den(z["x"], z["sigma"], **variant_kwargs(z, key)), z[key]), f"edge_{name}.{key}")
