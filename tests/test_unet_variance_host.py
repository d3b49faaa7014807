"""DenoiserWithVariance on the CPU: the oracle's float64 logvar, loss and gradients against the reference's recordings
(oracle/make_golden_unet_variance.py), the native loss's plumbing with the engine stubbed (which calls it makes, with which cotangents), the
refusals, the reference formula around a foreign inner model, and the argument checks of the new entry points, which need no GPU."""
import contextlib
import ctypes
import json
from pathlib import Path

import pytest
import torch
from torch import nn

import k_diffusion as K
from k_diffusion import _native

from conftest import load_npz, synth_sd
from oracle import kdiff_oracle as O

GOLDEN = Path(__file__).resolve().parent / "golden"
META = json.loads((GOLDEN / "unet_variance_meta.json").read_text())
CFG = {"model": {"type": "image_v1", "input_channels": 3, "input_size": [16, 16], "mapping_out": 32, "depths": [1, 2], "channels": [32, 64],
                 "self_attn_depths": [False, True], "mapping_cond_dim": 4, "augment_wrapper": True, "has_variance": True}}


def probe(shape, key):
    return torch.randn(shape, generator=torch.Generator().manual_seed(sum(map(ord, key))), dtype=torch.float64)


@pytest.mark.parametrize("name", sorted(META["cases"]))
def test_oracle_matches_the_reference(name):
    """unet_variance_oracle's float64 logvar, DenoiserWithVariance loss and every parameter's gradient (norm and probe) against the reference's"""
    from test_gpu_unet_variance import oracle_grads
    rec = load_npz("unet_variance.npz")
    cfg = META["configs"][name]
    model = K.config.make_model(K.config.load_config(cfg))
    inner = model.inner_model if isinstance(model, K.augmentation.KarrasAugmentWrapper) else model
    sd = synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, 3)
    kw = {k: rec[f"{name}_{k}"] for k in ("aug_cond", "mapping_cond") if f"{name}_{k}" in rec}
    x = rec[f"{name}_x"]
    loss, lv, grads = oracle_grads(cfg, sd, x, rec[f"{name}_noise"], rec[f"{name}_sigma"], kw, torch.ones(x.shape[0]), torch.float64)
    assert torch.allclose(loss, rec[f"{name}_loss_float64"].double(), rtol=1e-10, atol=0)
    assert torch.allclose(lv, rec[f"{name}_logvar_float64"].double(), rtol=1e-9, atol=1e-12)
    case = META["cases"][name]
    assert set(grads) == set(case)
    for k, g in grads.items():
        r = case[k]
        assert abs(g.norm().item() - r["norm"]) <= 1e-9 * r["norm"] + 1e-300, k
        assert abs((g * probe(g.shape, k)).sum().item() - r["probe"]) <= 1e-9 * r["norm"] * g.numel() ** 0.5 + 1e-300, k
    assert (grads["proj_out.weight"][-1] != 0).all() and grads["proj_out.bias"][-1] != 0


# ------------------------------------------------------------------------------------------------------------------------------
# plumbing with the engine stubbed
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def fake_cuda(monkeypatch):
    """CPU tensors that pass the device checks; the engine is replaced where a test needs one"""
    monkeypatch.setattr(_native, "require_cuda", lambda *t: None)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())


class _StubEngine:
    """F = 0.5 x and logvar = mean(x) per image; records each call"""
    cond_stride = 4

    def __init__(self, log):
        self.log = log

    def conditioning(self, sigma, *cond):
        return torch.zeros(sigma.shape[0], self.cond_stride)

    def forward_variance(self, x, sigma, cond, stride, sd, precision):
        self.log.append(("forward_variance", sd, precision))
        return 0.5 * x, x.flatten(1).mean(1)

    def train_forward(self, x, sigma, cond, stride, sd, precision):
        self.log.append(("train_forward", sd, precision))
        return 0.5 * x

    def forward_train(self, x, u, sigma, aug, cls, mc, cond, grads, precision=_native.PREC_FP32, dlogvar=None):
        self.log.append(("forward_train", precision, u.clone(), None if dlogvar is None else dlogvar.clone()))
        for g in grads.values():
            g.zero_()
        return 0.5 * x


def _stub_losses(monkeypatch):
    def variance_loss(x, noise, sigma, sd, f, lv):
        c_skip, c_out, _ = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sigma, sd)]
        r = f - (x - c_skip * (x + noise * sigma.view(-1, 1, 1, 1))) / c_out
        q = (r ** 2).flatten(1).mean(1) * torch.exp(-lv)
        return (q + lv) / 2, r * torch.exp(-lv).view(-1, 1, 1, 1) / r[0].numel(), (1 - q) / 2
    monkeypatch.setattr(_native, "loss_noised_input", lambda x, noise, sigma, sd: x + noise * sigma.view(-1, 1, 1, 1))
    monkeypatch.setattr(_native, "variance_loss", variance_loss)
    monkeypatch.setattr(_native, "denoiser_loss", lambda x, noise, sig, w, sd, f, kind: (f.flatten(1).mean(1), torch.ones_like(f)))
    return variance_loss


@pytest.mark.parametrize("wrapped", [True, False])
def test_native_loss_calls_and_cotangents(fake_cuda, monkeypatch, wrapped):
    """DenoiserWithVariance.loss: forward_variance at fp32 and the variance loss; the backward one forward_train whose u and dlogvar are the
    loss's cotangents times each sample's incoming gradient.  Denoiser.loss on the same model keeps train_forward and no dlogvar."""
    stub = _stub_losses(monkeypatch)
    cfg = K.config.load_config(CFG)
    outer = K.config.make_model(cfg)
    inner = outer.inner_model
    log = []
    monkeypatch.setattr(type(inner), "engine", lambda self, augment=False: _StubEngine(log))
    model = outer if wrapped else inner
    den = K.config.make_denoiser_wrapper(cfg)(model)
    assert type(den) is K.layers.DenoiserWithVariance and den._loss_kind == _native.LOSS_VARIANCE
    g = torch.Generator().manual_seed(0)
    x, noise = torch.randn(2, 3, 16, 16, generator=g), torch.randn(2, 3, 16, 16, generator=g)
    sig, mc, gw = torch.tensor([0.5, 2.0]), torch.randn(2, 4, generator=g), torch.tensor([1.5, -0.25])
    kw = dict(aug_cond=torch.zeros(2, 9), mapping_cond=mc) if wrapped else dict(mapping_cond=torch.cat([torch.zeros(2, 9), mc], 1))
    loss = den.loss(x, noise, sig, **kw)
    xin = x + noise * sig.view(-1, 1, 1, 1)
    want, cot, dlv = stub(x, noise, sig, cfg["model"]["sigma_data"], 0.5 * xin, xin.flatten(1).mean(1))
    assert torch.allclose(loss, want) and loss.grad_fn is not None
    (loss * gw).sum().backward()
    assert [c[:2] for c in log] == [("forward_variance", 0.0), ("forward_train", _native.PREC_FP32)]
    assert log[0][2] == _native.PREC_FP32
    assert torch.allclose(log[1][2], cot * gw.view(-1, 1, 1, 1)) and torch.allclose(log[1][3], dlv * gw)
    log.clear()
    K.layers.Denoiser(model, 0.5).loss(x, noise, sig, **kw).sum().backward()
    assert [c[0] for c in log] == ["train_forward", "forward_train"] and log[1][3] is None


def test_loss_refusals(fake_cuda):
    cfg = K.config.load_config(CFG)
    outer = K.config.make_model(cfg)
    den = K.config.make_denoiser_wrapper(cfg)(outer)
    x, sig, mc = torch.randn(2, 3, 16, 16), torch.tensor([0.5, 2.0]), torch.randn(2, 4)
    for i in range(3):
        args = [x, torch.randn_like(x), sig]
        args[i] = args[i].clone().requires_grad_()
        with pytest.raises(RuntimeError, match=("input", "noise", "sigma")[i]):
            den.loss(*args, mapping_cond=mc)
    outer.inner_model.dropout_rate = 0.05
    with pytest.raises(RuntimeError, match="dropout"):
        den.train().loss(x, torch.randn_like(x), sig, mapping_cond=mc)
    plain = K.config.make_model(K.config.load_config({"model": dict(CFG["model"], has_variance=False)}))
    for m in (plain, plain.inner_model):
        with pytest.raises(NotImplementedError, match="return_variance"):
            K.layers.DenoiserWithVariance(m, 0.5).loss(x, torch.randn_like(x), sig, mapping_cond=mc)
        with pytest.raises(NotImplementedError, match="has_variance"):
            m(x, sig, mapping_cond=mc, return_variance=True)


def test_transformers_and_cpu_tensors_refuse():
    x = torch.randn(1, 1, 8, 8)
    v1 = K.config.make_model(K.config.load_config({"model": {"type": "image_transformer_v1", "input_channels": 1, "input_size": [8, 8],
                                                             "patch_size": [2, 2], "depth": 1, "width": 64, "d_ff": 128}}))
    v2 = K.config.make_model(K.config.load_config(json.loads((GOLDEN / "cfg1_mnist_shapes.json").read_text())["config"]))
    for m in (v1, v2, K.augmentation.KarrasAugmentWrapper(v2)):
        with pytest.raises(NotImplementedError, match="return_variance"):
            K.layers.DenoiserWithVariance(m).loss(x, torch.randn_like(x), torch.ones(1))
    cfg = K.config.load_config(CFG)
    outer = K.config.make_model(cfg)
    x = torch.randn(1, 3, 16, 16)
    with pytest.raises(NotImplementedError, match="CUDA"):
        K.config.make_denoiser_wrapper(cfg)(outer).loss(x, torch.randn_like(x), torch.ones(1), mapping_cond=torch.zeros(1, 4))
    for m in (outer, outer.inner_model):
        with pytest.raises(NotImplementedError, match="fp32"):
            m.set_train_precision("tf32")


def test_foreign_inner_model_runs_the_reference_formula():
    class Inner(nn.Module):
        def __init__(self):
            super().__init__()
            self.w, self.v = nn.Parameter(torch.tensor(0.7)), nn.Parameter(torch.tensor(-0.3))

        def forward(self, x, sigma, return_variance=False):
            assert return_variance
            return x * self.w, self.v * sigma

    inner = Inner()
    x, noise, sig = torch.randn(3, 2, 4, 4), torch.randn(3, 2, 4, 4), torch.tensor([0.3, 1.0, 4.0])
    loss = K.layers.DenoiserWithVariance(inner, 0.5, weighting="snr", scales=2).loss(x, noise, sig)
    assert loss.shape == (3,) and loss.grad_fn is not None
    c_skip, c_out, c_in = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sig, 0.5)]
    noised = x + noise * sig.view(-1, 1, 1, 1)
    f, lv = noised * c_in * 0.7, (-0.3 * sig).view(-1, 1, 1, 1)
    want = (((f - (x - c_skip * noised) / c_out) ** 2 / torch.exp(lv) + lv) / 2).flatten(1).mean(1)
    assert torch.allclose(loss, want, rtol=1e-6)
    loss.sum().backward()
    assert inner.w.grad is not None and inner.v.grad is not None


# ------------------------------------------------------------------------------------------------------------------------------
# the new entry points' argument checks
# ------------------------------------------------------------------------------------------------------------------------------
def _handle(has_variance):
    cfg = K.config.load_config({"model": dict(CFG["model"], has_variance=has_variance)})
    outer = K.config.make_model(cfg)
    return _native.UNetEngine(outer.inner_model.engine_spec(True))


def test_entry_points_refuse_bad_arguments_without_a_gpu():
    L = _native.lib()
    p = ctypes.c_void_p(256)       # never dereferenced: every call below fails its checks first
    plain, var = _handle(False), _handle(True)
    fwd = lambda h, prec, logvar: L.kdb_unet_forward_variance(h._h, prec, 1, 16, 16, p, p, 0.0, p, 0, p, logvar, p, 1 << 20, None)
    assert fwd(plain, _native.PREC_FP32, p) == -1 and b"has_variance" in L.kdb_last_error()
    assert fwd(var, _native.PREC_FP32, None) == -1 and b"logvar" in L.kdb_last_error()
    assert fwd(var, _native.PREC_FP32, p) == -6                       # not finalized
    train = lambda h, prec, dlv: L.kdb_unet_forward_train_variance(h._h, prec, 1, 16, 16, p, p, None, None, p, 0, p, dlv, p, p, 1 << 20, None)
    assert train(plain, _native.PREC_FP32, p) == -1 and b"has_variance" in L.kdb_last_error()
    assert train(var, _native.PREC_FP32, None) == -1 and b"dlogvar" in L.kdb_last_error()
    assert train(var, _native.PREC_TF32, p) == -2 and b"fp32" in L.kdb_last_error()
    assert train(var, _native.PREC_FP32, p) == -6
    loss = lambda sd, lv, B: L.kdb_variance_loss(p, p, p, sd, p, lv, p, None, None, B, 16, None)
    assert loss(0.5, None, 1) == -1 and loss(0.0, p, 1) == -1 and loss(0.5, p, 0) == -1
    assert b"variance_loss" in L.kdb_last_error()
