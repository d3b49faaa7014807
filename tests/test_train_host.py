"""Training on the CPU side: the oracle's float64 loss and parameter gradients against the reference's (tests/golden/train*, recorded by
oracle/make_golden_train.py), param_groups against the reference's groups, and the refusals of Denoiser.loss."""
import contextlib
import ctypes
import json
from pathlib import Path

import numpy as np
import pytest
import torch
from torch import nn

from conftest import synth_sd
from oracle import kdiff_oracle as O

import k_diffusion as K

GOLDEN = Path(__file__).resolve().parent / "golden"
META = json.loads((GOLDEN / "train_meta.json").read_text())
NPZ = np.load(GOLDEN / "train.npz")
CLASS = {"model": {"type": "image_transformer_v2", "input_channels": 1, "input_size": [16, 16], "patch_size": [2, 2], "depths": [2, 1],
                   "widths": [32, 64], "d_ffs": [64, 96], "mapping_width": 64, "mapping_depth": 2, "mapping_d_ff": 96,
                   "loss_weighting": "soft-min-snr", "sigma_data": 0.6,
                   "self_attns": [{"type": "shifted-window", "d_head": 16, "window_size": 4}, {"type": "global", "d_head": 16}]},
         "dataset": {"num_classes": 10}}
LEVELS3 = {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [32, 32], "patch_size": [2, 2], "depths": [1, 1, 1],
                     "widths": [32, 48, 64], "d_ffs": [64, 96, 128], "mapping_width": 64, "mapping_depth": 1, "mapping_d_ff": 128,
                     "mapping_cond_dim": 12, "sigma_data": 0.5,
                     "self_attns": [{"type": "shifted-window", "d_head": 16, "window_size": 4}, {"type": "global", "d_head": 16},
                                    {"type": "none"}]}}
# the reference's transformer configs as recorded beside their parameter shapes: cfg1 (MNIST) and the CIFAR-10 transformer
REF_CONFIGS = {"cfg1": "cfg1_mnist_shapes.json", "cifar10": "cifar10_transformer_shapes.json"}
CASES = {"class": (CLASS, False), "class_simple": (CLASS, True), "levels3": (LEVELS3, False),
         **{name: (json.loads((GOLDEN / f).read_text())["config"], False) for name, f in REF_CONFIGS.items()}}
BUFFERS = ("pos_emb.freqs", "time_emb.weight", "aug_emb.weight")


def model_of(cfg):
    cfg = K.config.load_config(json.loads(json.dumps(cfg)))
    inner = K.config.make_model(cfg)
    return cfg, inner, synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, 3)


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_loss_and_gradients_match_the_reference(case):
    cfg, simple = CASES[case]
    cfg, _, sd = model_of(cfg)
    m = cfg["model"]
    p = {k: v.double().requires_grad_(not k.endswith(BUFFERS)) for k, v in sd.items()}
    x, noise, sigma = (torch.from_numpy(NPZ[f"{case}_{k}"]).double() for k in ("x", "noise", "sigma"))
    kw = {}
    if cfg["dataset"]["num_classes"]:
        kw["class_cond"] = torch.tensor([3, 3])
    if m["mapping_cond_dim"]:   # make_golden_train's inputs draw aug_cond and mapping_cond after sigma from one generator
        g = torch.Generator().manual_seed(11)
        for t in (x, noise, sigma):
            torch.randn(t.shape, generator=g)
        kw["mapping_cond"] = torch.cat([torch.randn(2, 9, generator=g) * 0.3, torch.randn(2, m["mapping_cond_dim"] - 9, generator=g)], 1).double()
    sdat = m["sigma_data"]
    c_skip, c_out, c_in = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sigma, sdat)]
    s4 = sigma.view(-1, 1, 1, 1)
    noised = x + noise * s4
    f = O.model_forward(p, m, noised * c_in, sigma, **kw)
    if simple:
        loss = (((noised - (f * c_out + noised * c_skip)) / s4 - noise) ** 2).flatten(1).mean(1)
    else:
        w = (sigma * sdat) ** 2 / (sigma ** 2 + sdat ** 2) ** 2 if m["loss_weighting"] == "soft-min-snr" else torch.ones_like(sigma)
        loss = ((f - (x - c_skip * noised) / c_out) ** 2).flatten(1).mean(1) * w
    np.testing.assert_allclose(loss.detach().numpy(), NPZ[f"{case}_loss_float64"], rtol=1e-7)
    loss.sum().backward()
    want = META["cases"][case]   # the reference and the oracle agree to ~1e-6 relative in float64 (their op orders differ)
    assert set(want) == {k for k, t in p.items() if t.requires_grad}
    for k, w in want.items():
        g = p[k].grad
        assert g.norm().item() == pytest.approx(w["norm"], rel=2e-5), k
        probe = torch.randn(g.shape, generator=torch.Generator().manual_seed(sum(map(ord, k))), dtype=torch.float64)
        assert (g * probe).sum().item() == pytest.approx(w["probe"], rel=2e-5, abs=2e-5 * w["norm"]), k


@pytest.mark.parametrize("case", ["class", "levels3", "cfg1", "cifar10"])
def test_param_groups_match_the_reference(case):
    _, inner, _ = model_of(CASES[case][0])
    groups = inner.param_groups(1e-3, 0.25)
    names = {id(p): k for k, p in inner.named_parameters()}
    assert [[names[id(p)] for p in g["params"]] for g in groups] == META["param_groups"][case]
    assert [g["lr"] for g in groups] == [1e-3, 1e-3, 2.5e-4, 2.5e-4]
    assert [g.get("weight_decay") for g in groups] == [None, 0.0, None, 0.0]
    wrapped = K.augmentation.KarrasAugmentWrapper(inner).param_groups(1e-3, 0.25)
    assert [[names[id(p)] for p in g["params"]] for g in wrapped] == META["param_groups"][case]


@pytest.fixture
def cpu_native(monkeypatch):
    from k_diffusion import _native
    monkeypatch.setattr(_native, "require_cuda", lambda *t: None)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())


def test_loss_refusals(cpu_native):
    cfg, inner, sd = model_of(CLASS)
    inner.load_state_dict(sd)
    x = torch.randn(2, 1, 16, 16)
    sig, cc = torch.tensor([0.5, 2.0]), torch.tensor([1, 2])
    with pytest.raises(NotImplementedError, match="DCT"):
        K.layers.Denoiser(inner, 0.6, scales=2).loss(x, torch.randn_like(x), sig, class_cond=cc)
    with pytest.raises(NotImplementedError, match="return_variance"):
        K.layers.DenoiserWithVariance(inner, 0.6).loss(x, torch.randn_like(x), sig, class_cond=cc)
    model = K.config.make_denoiser_wrapper(cfg)(inner)
    for i in range(3):
        args = [x, torch.randn_like(x), sig]
        args[i] = args[i].clone().requires_grad_()
        with pytest.raises(RuntimeError, match=("input", "noise", "sigma")[i]):
            model.loss(*args, class_cond=cc)
    inner.levels[0].dropout = 0.1
    with pytest.raises(RuntimeError, match="dropout"):
        model.train().loss(x, torch.randn_like(x), sig, class_cond=cc)
    with pytest.raises(ValueError, match="class_cond"):
        model.eval().loss(x, torch.randn_like(x), sig)


def test_v1_and_unet_loss_raise(cpu_native):
    v1 = K.config.make_model(K.config.load_config({"model": {"type": "image_transformer_v1", "input_channels": 1, "input_size": [8, 8],
                                                             "patch_size": [2, 2], "depth": 1, "width": 64, "d_ff": 128}}))
    x = torch.randn(1, 1, 8, 8)
    with pytest.raises(NotImplementedError, match="image_transformer_v2"):
        K.layers.Denoiser(v1).loss(x, torch.randn_like(x), torch.ones(1))
    ucfg = K.config.load_config({"model": {"type": "image_v1", "input_channels": 3, "input_size": [16, 16], "mapping_out": 32,
                                           "depths": [1, 1], "channels": [32, 64], "self_attn_depths": [False, True]}})
    unet = K.config.make_model(ucfg)
    x = torch.randn(1, 3, 16, 16)
    with pytest.raises(NotImplementedError):
        K.layers.Denoiser(unet).loss(x, torch.randn_like(x), torch.ones(1))


def test_foreign_inner_model_loss_is_the_reference_formula():
    class Inner(nn.Module):
        def __init__(self):
            super().__init__()
            self.w = nn.Parameter(torch.tensor(0.7))

        def forward(self, x, sigma):
            return x * self.w

    inner = Inner()
    x, noise, sig = torch.randn(3, 2, 4, 4), torch.randn(3, 2, 4, 4), torch.tensor([0.3, 1.0, 4.0])
    for cls, weighting in ((K.layers.Denoiser, "snr"), (K.layers.SimpleLossDenoiser, "karras")):
        loss = cls(inner, 0.5, weighting=weighting).loss(x, noise, sig)
        assert loss.shape == (3,) and loss.grad_fn is not None
        c_skip, c_out, c_in = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sig, 0.5)]
        noised = x + noise * sig.view(-1, 1, 1, 1)
        if cls is K.layers.Denoiser:
            want = ((noised * c_in * inner.w - (x - c_skip * noised) / c_out) ** 2).flatten(1).mean(1) * (0.25 / (sig ** 2 + 0.25))
        else:
            den = noised * c_in * inner.w * c_out + noised * c_skip
            want = (((noised - den) / sig.view(-1, 1, 1, 1) - noise) ** 2).flatten(1).mean(1)
        assert torch.allclose(loss, want, rtol=1e-5)


def test_v1_param_groups_still_raise():
    v1 = K.config.make_model(K.config.load_config({"model": {"type": "image_transformer_v1", "input_channels": 1, "input_size": [8, 8],
                                                             "patch_size": [2, 2], "depth": 1, "width": 64, "d_ff": 128}}))
    with pytest.raises(NotImplementedError, match="image_transformer_v1"):
        v1.param_groups(1e-3)
    with pytest.raises(NotImplementedError, match="image_transformer_v1"):
        K.augmentation.KarrasAugmentWrapper(v1).param_groups(1e-3)


def test_set_grad_checks_key_shape_and_buffers_without_gpu():
    from k_diffusion import _native
    L = _native.lib()
    _, inner, _ = model_of(CLASS)
    eng_cfg = _native.Engine._config(inner.engine_spec())
    h = ctypes.c_void_p()
    assert L.kdb_model_create(ctypes.byref(eng_cfg), ctypes.byref(h)) == 0
    try:
        host = torch.zeros(4)   # set_tensor / set_grad only record the pointer: a host address suffices for the checks
        dims = lambda *s: (ctypes.c_int64 * len(s))(*s)
        for key, shape in (("time_emb.weight", (32, 1)), ("out_norm.scale", (32,))):
            assert L.kdb_model_set_tensor(h, key.encode(), _native.ptr(host), dims(*shape), len(shape)) == 0
        assert L.kdb_model_set_grad(h, b"out_norm.scale", _native.ptr(host), dims(32), 1) == 0
        assert L.kdb_model_set_grad(h, b"out_norm.scale", None, None, 0) == 0        # unbinds
        assert L.kdb_model_set_grad(h, b"no.such.key", _native.ptr(host), dims(32), 1) == -3     # KDB_ERR_MISSING_KEY
        assert b"no.such.key" in L.kdb_last_error()
        assert L.kdb_model_set_grad(h, b"out_norm.scale", _native.ptr(host), dims(33), 1) == -4  # KDB_ERR_BAD_SHAPE
        assert L.kdb_model_set_grad(h, b"time_emb.weight", _native.ptr(host), dims(32, 1), 2) == -1   # KDB_ERR_BAD_ARG: a buffer
        assert b"buffer" in L.kdb_last_error()
    finally:
        L.kdb_model_destroy(h)


def test_reduction_wrappers_refuse_mismatched_operands(cpu_native, monkeypatch):
    """The C reductions take no operand extents: each wrapper checks them before the call, so a mismatch raises instead of reading or
    writing out of bounds"""
    from k_diffusion import _native
    monkeypatch.setattr(_native, "lib", lambda: pytest.fail("reached the library"))
    z = torch.zeros
    bad = [
        lambda: _native.wgrad(z(10, 4), z(9, 5)),                                           # fewer x rows than dy rows
        lambda: _native.wgrad(z(10, 4), z(10, 5), out=z(5, 4)),
        lambda: _native.wgrad(z(10, 4), z(10, 5).t().contiguous().t()),                     # x columns not contiguous
        lambda: _native.wgrad_patch_in(z(2 * 7 * 7, 8), z(2, 1, 28, 28), (4, 3)),            # 28 is not a multiple of 3
        lambda: _native.wgrad_patch_in(z(2 * 7 * 6, 8), z(2, 1, 28, 28), (4, 4)),            # one token row per patch
        lambda: _native.wgrad_patch_out(z(1, 3, 8, 8), z(16, 32), z(32), z(15), (2, 2)),     # rstd per token
        lambda: _native.wgrad_patch_out(z(1, 3, 8, 8), z(16, 32), z(31), z(16), (2, 2)),     # scale per channel
        lambda: _native.norm_scale_grad(z(10, 8), z(10, 8), 3),                              # rows a multiple of the rows per image
        lambda: _native.norm_scale_grad(z(10, 8), z(10, 9)),
        lambda: _native.norm_scale_grad(z(10, 8), z(10, 8), 5, out=z(8 + 8), ldo=7),         # images overlap
        lambda: _native.norm_scale_grad(z(10, 8), z(10, 8), 5, out=z(10 + 7), ldo=10),       # too short for two images 10 apart
        lambda: _native.colsum(z(10, 4).t()),
        lambda: _native.colsum(z(10, 4), out=z(5)),
        lambda: _native.split_fac_grad(z(1, 2, 2, 12), z(1, 4, 4, 3), z(1, 4, 5, 3)),
        lambda: _native.split_fac_grad(z(1, 2, 3, 12), z(1, 4, 5, 3), z(1, 4, 5, 3)),      # odd fine grid
        lambda: _native.class_emb_grad(z(4, 8), torch.zeros(4, dtype=torch.int32), 11),
        lambda: _native.class_emb_grad(z(4, 8), torch.zeros(3, dtype=torch.int64), 11),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(ValueError):
            call()
            pytest.fail(f"case {i} was accepted")
