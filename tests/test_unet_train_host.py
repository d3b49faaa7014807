"""The U-Net's training front end on the CPU: param_groups against the reference's rule, and the refusals of Denoiser.loss around it, which
come before any engine is built."""
import contextlib

import pytest
import torch

import k_diffusion as K
from k_diffusion import _native

CFG = {"model": {"type": "image_v1", "input_channels": 3, "input_size": [16, 16], "mapping_out": 32, "depths": [1, 2], "channels": [32, 64],
                 "self_attn_depths": [False, True], "mapping_cond_dim": 4, "augment_wrapper": True}}


def model():
    cfg = K.config.load_config(CFG)
    wrapped = K.config.make_model(cfg)
    return cfg, wrapped, wrapped.inner_model


def test_param_groups_follow_the_reference_rule():
    """Weight decay for the weights named mapping* or u_net*, none for everything else; every parameter in exactly one group"""
    _, wrapped, inner = model()
    names = {id(p): k for k, p in inner.named_parameters()}
    for groups in (inner.param_groups(1e-3), wrapped.param_groups(1e-3)):
        wd, no_wd = ([names[id(p)] for p in g["params"]] for g in groups)
        assert [g["lr"] for g in groups] == [1e-3, 1e-3] and groups[1]["weight_decay"] == 0.0 and "weight_decay" not in groups[0]
        assert sorted(wd + no_wd) == sorted(names.values())
        assert all(k.startswith(("mapping", "u_net")) and k.endswith(".weight") for k in wd)
        assert all(not (k.startswith(("mapping", "u_net")) and k.endswith(".weight")) for k in no_wd)
        assert "mapping_cond.weight" in wd and "u_net.d_blocks.0.1.main.0.mapper.weight" in wd
        assert "proj_in.weight" in no_wd and "u_net.d_blocks.0.1.main.0.mapper.bias" in no_wd
    assert inner.param_groups()[0]["lr"] == 2e-4


@pytest.fixture
def fake_cuda(monkeypatch):
    """CPU tensors that pass the U-Net loss's device check; the engine is never reached"""
    monkeypatch.setattr(_native, "require_cuda", lambda *t: None)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())


def test_loss_refusals(fake_cuda):
    cfg, wrapped, inner = model()
    x, sig, mc = torch.randn(2, 3, 16, 16), torch.tensor([0.5, 2.0]), torch.randn(2, 4)
    with pytest.raises(NotImplementedError, match="DCT"):
        K.layers.Denoiser(wrapped, 0.5, scales=2).loss(x, torch.randn_like(x), sig, mapping_cond=mc)
    den = K.config.make_denoiser_wrapper(cfg)(wrapped)
    for i in range(3):
        args = [x, torch.randn_like(x), sig]
        args[i] = args[i].clone().requires_grad_()
        with pytest.raises(RuntimeError, match=("input", "noise", "sigma")[i]):
            den.loss(*args, mapping_cond=mc)
    inner.dropout_rate = 0.05
    with pytest.raises(RuntimeError, match="dropout"):
        den.train().loss(x, torch.randn_like(x), sig, mapping_cond=mc)


def test_cpu_tensors_and_tf32_training_raise_not_implemented():
    _, wrapped, inner = model()
    x = torch.randn(1, 3, 16, 16)
    with pytest.raises(NotImplementedError, match="CUDA"):
        K.layers.Denoiser(wrapped).loss(x, torch.randn_like(x), torch.ones(1), mapping_cond=torch.zeros(1, 4))
    for m in (inner, wrapped):
        with pytest.raises(NotImplementedError, match="fp32"):
            m.set_train_precision("tf32")


# ------------------------------------------------------------------------------------------------------------------------------
# the oracle's float64 autograd and param_groups against the reference's recordings (oracle/make_golden_unet_train.py)
# ------------------------------------------------------------------------------------------------------------------------------
import json  # noqa: E402
from pathlib import Path  # noqa: E402

from conftest import load_npz, synth_sd  # noqa: E402
from test_gpu_unet_train import oracle_grads  # noqa: E402

GOLDEN = Path(__file__).resolve().parent / "golden"
META = json.loads((GOLDEN / "unet_train_meta.json").read_text())
REC = load_npz("unet_train.npz")


def probe(shape, key):
    return torch.randn(shape, generator=torch.Generator().manual_seed(sum(map(ord, key))), dtype=torch.float64)


def recorded_case(name):
    cfg = META["configs"][name]
    kw = {k: REC[f"{name}_{k}"] for k in ("aug_cond", "mapping_cond") if f"{name}_{k}" in REC}
    return cfg, REC[f"{name}_x"], REC[f"{name}_noise"], REC[f"{name}_sigma"], kw


@pytest.mark.parametrize("name", sorted(META["cases"]))
def test_oracle_gradients_match_the_reference(name):
    """unet_oracle's float64 loss and every parameter's float64 gradient (norm and probe) against the reference's Denoiser.loss"""
    cfg, x, noise, sigma, kw = recorded_case(name)
    model = K.config.make_model(K.config.load_config(cfg))
    inner = model.inner_model if isinstance(model, K.augmentation.KarrasAugmentWrapper) else model
    sd = synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, 3)
    loss, grads = oracle_grads(cfg, sd, x, noise, sigma, kw, torch.ones(x.shape[0]), torch.float64)
    assert torch.allclose(loss, REC[f"{name}_loss_float64"].double(), rtol=1e-10, atol=0)
    rec = META["cases"][name]
    assert set(grads) == set(rec) and not META["no_grad"][name]
    for k, g in grads.items():
        r = rec[k]
        assert abs(g.norm().item() - r["norm"]) <= 1e-9 * r["norm"] + 1e-300, k
        assert abs((g * probe(g.shape, k)).sum().item() - r["probe"]) <= 1e-9 * r["norm"] * g.numel() ** 0.5 + 1e-300, k
    if cfg["model"]["has_variance"]:
        assert rec["proj_out.bias"]["norm"] > 0 and (grads["proj_out.weight"][-1] == 0).all() and grads["proj_out.bias"][-1] == 0


@pytest.mark.parametrize("name", sorted(META["param_groups"]))
def test_param_groups_match_the_reference(name):
    model = K.config.make_model(K.config.load_config(META["configs"][name]))
    names = {id(p): k for k, p in model.named_parameters()}
    names = {i: k[len("inner_model."):] if k.startswith("inner_model.") else k for i, k in names.items()}
    assert [[names[id(p)] for p in g["params"]] for g in model.param_groups()] == META["param_groups"][name]
