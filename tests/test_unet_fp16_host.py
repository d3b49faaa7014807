"""The fp16 precision on the CPU: how set_precision, KDB200_PRECISION and the augment wrapper select it for the image_v1 U-Net, that
auto never means fp16 (not even for fp16 parameters), that bf16 is still refused and the transformer refuses fp16, the fp16
restatement the GPU tests hold the engine to, and that the oracle with that restatement reproduces the reference's fp16 deviation
recorded in tests/golden/fp16_budget.json."""
import json

import pytest
import torch

import k_diffusion as K
from conftest import GOLDEN, load_npz
from oracle import kdiff_oracle as O
from oracle import unet_oracle as U
from oracle.fixtures import synth_sd
from oracle.make_golden_fp16 import f16_round
from test_unet_edges_host import VARIANTS, variant_kwargs
from test_unet_tf32_host import transformer, unet

META = json.loads((GOLDEN / "unet_configs.json").read_text())
EDGES = json.loads((GOLDEN / "unet_edges.json").read_text())
BUDGET = json.loads((GOLDEN / "fp16_budget.json").read_text())
N = K._native


def test_set_precision_selects_fp16_directly_and_through_the_augment_wrapper(monkeypatch):
    monkeypatch.delenv("KDB200_PRECISION", raising=False)
    model = unet()
    assert isinstance(model, K.augmentation.KarrasAugmentWrapper)
    assert N.PREC_FP16 == 3
    for name in ("fp16", "float16"):
        assert model.set_precision(name) is model
        assert model.resolved_precision() == model.inner_model.resolved_precision() == N.PREC_FP16
    assert model.inner_model.set_precision("tf32").resolved_precision() == N.PREC_TF32
    assert model.inner_model.set_precision("fp16").resolved_precision() == N.PREC_FP16
    assert model.resolved_precision() == N.PREC_FP16
    for auto in (None, "auto"):
        assert model.set_precision(auto).resolved_precision() == N.PREC_FP32
    for bad in ("bf16", "bfloat16", "half16"):
        with pytest.raises(ValueError):
            model.set_precision(bad)


def test_environment_selects_fp16_unless_the_model_says_otherwise(monkeypatch):
    model = unet()
    monkeypatch.setenv("KDB200_PRECISION", "fp16")
    assert model.resolved_precision() == N.PREC_FP16
    assert model.set_precision("tf32").resolved_precision() == N.PREC_TF32
    assert model.set_precision("fp32").resolved_precision() == N.PREC_FP32
    monkeypatch.setenv("KDB200_PRECISION", "float16")
    assert model.set_precision(None).resolved_precision() == N.PREC_FP16
    monkeypatch.setenv("KDB200_PRECISION", "auto")
    assert model.resolved_precision() == N.PREC_FP32
    monkeypatch.setenv("KDB200_PRECISION", "bf16")
    with pytest.raises(ValueError):
        model.resolved_precision()


def test_auto_never_resolves_to_fp16(monkeypatch):
    monkeypatch.delenv("KDB200_PRECISION", raising=False)
    assert K.models.flags.resolve_precision(None, torch.float16) == "fp32"
    assert K.models.flags.resolve_precision("auto", torch.float16) == "fp32"
    assert K.models.flags.resolve_precision("fp16", torch.float32) == "fp16"
    model = unet().half()
    assert next(model.parameters()).dtype == torch.float16
    assert model.set_precision(None).resolved_precision() == N.PREC_FP32
    with torch.autocast("cpu", dtype=torch.float16):
        assert model.resolved_precision() == N.PREC_FP32


def test_transformer_refuses_fp16(monkeypatch):
    monkeypatch.delenv("KDB200_PRECISION", raising=False)
    inner = transformer()
    with pytest.raises(ValueError, match="fp16"):
        inner.set_precision("fp16").resolved_precision()
    inner.set_precision(None)
    assert inner.resolved_precision() == N.PREC_FP32
    monkeypatch.setenv("KDB200_PRECISION", "fp16")
    with pytest.raises(ValueError, match="fp16"):
        inner.resolved_precision()


def test_fp16_restatement():
    """the restatement of the engine's operand rounding (oracle/make_golden_fp16.py): nearest, ties to even, by way of fp32, inf past the
    largest finite fp16"""
    ulp = 2.0 ** -10
    x = torch.tensor([1 + ulp / 2, 1 + ulp / 2 + 2.0 ** -20, 1 + 1.5 * ulp, -(1 + ulp / 2), 1 + ulp * 0.49, 3.0, 65519.0, 65520.0, -65520.0,
                      2.0 ** -25, 2.0 ** -25 + 2.0 ** -40], dtype=torch.float64)
    assert f16_round(x).tolist() == [1.0, 1 + ulp, 1 + 2 * ulp, -1.0, 1.0, 3.0, 65504.0, float("inf"), float("-inf"), 0.0, 2.0 ** -24]


def reproduced(monkeypatch, sd, mcfg):
    """the oracle's denoiser (fp32) with every Conv2d and the attention at fp16, as oracle/make_golden_fp16.py runs the reference"""
    from test_gpu_unet_fp16 import F16Functional
    monkeypatch.setattr(U, "F", F16Functional([]))
    return U.make_denoiser(sd, mcfg)


def close_to_budget(got, key):
    """the oracle and the reference differ by fp32 noise, which moves a few operands across an fp16 boundary: 10% of the deviation"""
    assert abs(got - BUDGET[key]) <= 0.1 * BUDGET[key], f"{key}: oracle {got:.4e} vs recorded {BUDGET[key]:.4e}"


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("name", sorted(META))
def test_oracle_reproduces_the_recorded_fp16_budget(name, monkeypatch):
    z = load_npz(f"unet_{name}.npz")
    den = reproduced(monkeypatch, U.strip_prefix(synth_sd(META[name]["shapes"], 1)), META[name]["config"]["model"])
    with torch.no_grad():
        close_to_budget(rel_l2(den(z["x"], z["sigma"]), z["denoised"]), f"{name}.denoised")
        close_to_budget(rel_l2(den(z["x"], z["sigma"], aug_cond=z["aug_cond"]), z["denoised_aug"]), f"{name}.denoised_aug")
        if name == "mnist":
            close_to_budget(rel_l2(O.sample_heun(den, z["heun_x"], z["heun_sigmas"]), z["heun"]), "mnist.heun10")


@pytest.mark.parametrize("name", sorted(EDGES))
def test_oracle_reproduces_the_recorded_fp16_budget_of_the_edge_configs(name, monkeypatch):
    z = load_npz(f"unet_edge_{name}.npz")
    den = reproduced(monkeypatch, U.strip_prefix(synth_sd(EDGES[name]["shapes"], 1)), EDGES[name]["config"]["model"])
    with torch.no_grad():
        for key in (k for k in VARIANTS if k in z):
            close_to_budget(rel_l2(den(z["x"], z["sigma"], **variant_kwargs(z, key)), z[key]), f"edge_{name}.{key}")
