"""The tf32 training precision of image_transformer_v2 on the CPU side: set_train_precision's values and refusals, which engine calls the
loss makes at each precision (a stubbed engine), and the tf32 restatement of a training step that the GPU tests (tests/test_gpu_train_tf32.py)
hold the engine to: every token-stream Linear (qkv, out, up, down, merge and split projections) with its activation truncated to tf32 and its
weight rounded, in the forward; the output gradient truncated and the weight rounded in the input gradient; both operands truncated in the
weight gradient.  Everything else is the oracle's exact arithmetic."""
import contextlib
import json

import pytest
import torch
from torch.overrides import TorchFunctionMode

from conftest import synth_sd
from oracle import kdiff_oracle as O
from oracle.make_golden_tf32 import tf32_round, tf32_trunc

import k_diffusion as K
from k_diffusion import _native

CLASS = {"model": {"type": "image_transformer_v2", "input_channels": 1, "input_size": [16, 16], "patch_size": [2, 2], "depths": [2, 1],
                   "widths": [32, 64], "d_ffs": [64, 96], "mapping_width": 64, "mapping_depth": 2, "mapping_d_ff": 96,
                   "loss_weighting": "soft-min-snr", "sigma_data": 0.6,
                   "self_attns": [{"type": "shifted-window", "d_head": 16, "window_size": 4}, {"type": "global", "d_head": 16}]},
         "dataset": {"num_classes": 10}}
BUFFERS = ("pos_emb.freqs", "time_emb.weight", "aug_emb.weight")


def token_stream_keys(keys):
    """the state-dict keys of the token-stream Linears (the mapping network's up_proj / down_proj are not among them)"""
    return {k for k in keys if k.endswith(("self_attn.qkv_proj.weight", "self_attn.out_proj.weight", "ff.up_proj.weight", "ff.down_proj.weight"))
            or (k.startswith(("merges.", "splits.")) and k.endswith(".proj.weight"))}


class _Tf32Linear(torch.autograd.Function):
    """y = a w^T with the operands the engine's tf32 route gives the tensor cores; products and sums in a's dtype"""

    @staticmethod
    def forward(ctx, a, w):
        ctx.save_for_backward(a, w)
        return tf32_trunc(a) @ tf32_round(w).T

    @staticmethod
    def backward(ctx, g):
        a, w = ctx.saved_tensors
        gt = tf32_trunc(g)
        dw = gt.reshape(-1, g.shape[-1]).T @ tf32_trunc(a).reshape(-1, a.shape[-1])
        return gt @ tf32_round(w), dw


_MATMULS = (torch.Tensor.__matmul__, torch.Tensor.matmul, torch.matmul)


class Tf32Linears(TorchFunctionMode):
    """Every `x @ w.T` whose w is one of `weights` (the oracle's form of an nn.Linear) runs as _Tf32Linear; `hit` collects the ids of the
    weights it rewrote, so a caller can check that no token-stream Linear escaped as exact arithmetic"""

    def __init__(self, weights):
        super().__init__()
        self.ids = {id(w) for w in weights}
        self.hit = set()

    def __torch_function__(self, func, types, args=(), kwargs=None):
        if func in _MATMULS and len(args) == 2 and not kwargs:
            a, b = args
            base = b._base
            if base is not None and id(base) in self.ids and b.ndim == 2 and tuple(b.shape) == tuple(base.shape[::-1]):
                self.hit.add(id(base))
                return _Tf32Linear.apply(a, base)
        return func(*args, **(kwargs or {}))


def restated_grads(cfg, sd, x, noise, sigma, kw, gw, dtype, tf32, simple=False):
    """(losses, {key: gradient}) of sum(loss * gw) for the oracle's model around layers.py:76-86 (or :107-111) in `dtype`, with the
    token-stream Linears at tf32 when `tf32`.  kw: class_cond, or aug_cond and mapping_cond (the augment wrapper's concatenation)."""
    m = cfg["model"]
    params = {k: v.detach().to(dtype, copy=True).requires_grad_(not k.endswith(BUFFERS)) for k, v in sd.items()}
    x, noise, sigma, gw = x.to(dtype), noise.to(dtype), sigma.to(dtype), gw.to(dtype)
    kw = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in kw.items()}
    if "aug_cond" in kw:
        kw["mapping_cond"] = torch.cat([kw.pop("aug_cond"), kw["mapping_cond"]], 1)
    sd_ = m["sigma_data"]
    c_skip, c_out, c_in = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sigma, sd_)]
    s4 = sigma.view(-1, 1, 1, 1)
    noised = x + noise * s4
    mode = Tf32Linears([params[k] for k in token_stream_keys(params)]) if tf32 else contextlib.nullcontext()
    with mode as seen:
        f = O.model_forward(params, m, noised * c_in, sigma, **kw)
        if simple:
            loss = (((noised - (f * c_out + noised * c_skip)) / s4 - noise) ** 2).flatten(1).mean(1)
        else:
            w = (sigma * sd_) ** 2 / (sigma ** 2 + sd_ ** 2) ** 2 if m["loss_weighting"] == "soft-min-snr" else torch.ones_like(sigma)
            loss = ((f - (x - c_skip * noised) / c_out) ** 2).flatten(1).mean(1) * w
        (loss * gw).sum().backward()
    if tf32:
        missed = sorted(k for k in token_stream_keys(params) if id(params[k]) not in seen.hit)
        assert not missed, f"token-stream Linears the restatement left exact: {missed}"
    return loss.detach(), {k: p.grad for k, p in params.items() if p.requires_grad}


def model_of(cfg):
    cfg = K.config.load_config(json.loads(json.dumps(cfg)))
    inner = K.config.make_model(cfg)
    return cfg, inner, synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, 3)


def test_set_train_precision_values_and_refusals():
    cfg, inner, _ = model_of(CLASS)
    assert getattr(inner, "train_precision", _native.PREC_FP32) == _native.PREC_FP32
    for p, code in (("tf32", _native.PREC_TF32), ("fp32", _native.PREC_FP32), ("tf32", _native.PREC_TF32), ("float32", _native.PREC_FP32),
                    ("tf32", _native.PREC_TF32), (None, _native.PREC_FP32)):
        assert inner.set_train_precision(p) is inner
        assert inner.train_precision == code
    for bad in ("bf16", "fp16", "auto", "TF32", 32, ["tf32"], {"tf32": 1}, 2.5):
        with pytest.raises(ValueError):
            inner.set_train_precision(bad)
    wrapped = K.augmentation.KarrasAugmentWrapper(inner)
    assert wrapped.set_train_precision("tf32") is wrapped and inner.train_precision == _native.PREC_TF32
    # the sampling precision and its refusal of tf32 are untouched
    assert inner.set_precision("bf16").precision == "bf16"
    inner.set_precision("tf32")
    with pytest.raises(ValueError, match="image_v1 U-Net"):
        inner.resolved_precision()


def test_v1_and_unet_have_no_training_precision():
    v1 = K.config.make_model(K.config.load_config({"model": {"type": "image_transformer_v1", "input_channels": 1, "input_size": [8, 8],
                                                             "patch_size": [2, 2], "depth": 1, "width": 64, "d_ff": 128}}))
    unet = K.config.make_model(K.config.load_config({"model": {"type": "image_v1", "input_channels": 3, "input_size": [16, 16],
                                                               "mapping_out": 32, "depths": [1, 1], "channels": [32, 64],
                                                               "self_attn_depths": [False, True]}}))
    for m in (v1, unet, K.augmentation.KarrasAugmentWrapper(unet), K.augmentation.KarrasAugmentWrapper(v1)):
        for p in ("tf32", "fp32"):
            with pytest.raises(NotImplementedError):
                m.set_train_precision(p)


def test_training_calls_refuse_precisions_without_gpu():
    """The training calls' refusals of a precision need no GPU and no finalize: a bad value, the v1 family, widths the tensor-core GEMM
    cannot stream; a precision they accept meets the finalize check"""
    L = _native.lib()

    def calls(h, precision):   # kdb_model_forward_train, then kdb_model_train_forward, with every other argument NULL or zero
        yield L.kdb_model_forward_train(h, precision, 1, 16, 16, None, None, None, None, None, None, 0, None, None, None, None, 0, None)
        yield L.kdb_model_train_forward(h, precision, 1, 16, 16, None, None, 0.0, None, 0, None, None, 0, None)

    _, inner, _ = model_of(CLASS)
    eng = _native.Engine(inner.engine_spec())
    for good in (_native.PREC_TF32, _native.PREC_FP32):
        assert tuple(calls(eng._h, good)) == (-6, -6)   # KDB_ERR_NOT_FINAL
    for bad in (_native.PREC_BF16, _native.PREC_FP16, 7):
        assert tuple(calls(eng._h, bad)) == (-2, -2)   # KDB_ERR_UNSUPPORTED
    odd = inner.engine_spec()
    odd["levels"][0]["d_ff"] = 66
    odd_eng = _native.Engine(odd)
    for rc in calls(odd_eng._h, _native.PREC_TF32):
        assert rc == -2 and b"multiples of 4" in L.kdb_last_error()
    assert tuple(calls(odd_eng._h, _native.PREC_FP32)) == (-6, -6)
    v1 = K.config.make_model(K.config.load_config({"model": {"type": "image_transformer_v1", "input_channels": 1, "input_size": [8, 8],
                                                             "patch_size": [2, 2], "depth": 1, "width": 64, "d_ff": 128}}))
    v1eng = _native.Engine(v1.engine_spec())
    for p in (_native.PREC_FP32, _native.PREC_TF32):
        assert tuple(calls(v1eng._h, p)) == (-2, -2)


class _StubEngine:
    """The Engine calls of Denoiser.loss, recorded; values are zeros"""

    def __init__(self, log):
        self.log, self.cond_stride = log, 4

    def conditioning(self, sigma, *args):
        self.log.append("conditioning")
        return torch.zeros(sigma.shape[0], 4)

    def forward(self, x, sigma, cond, stride, sigma_data, precision, out=None):
        self.log.append(("forward", precision))
        return torch.zeros_like(x)

    def train_forward(self, x, sigma, cond, stride, sigma_data, precision, out=None):
        self.log.append(("train_forward", sigma_data, precision))
        return torch.zeros_like(x)

    def forward_train(self, x, u, sigma, aug, cls, mc, cond, grads, out=None, grad_x=None, precision=_native.PREC_FP32):
        self.log.append(("forward_train", precision))
        for g in grads.values():
            g.zero_()
        return torch.zeros_like(x)

    def check_class_range(self, class_cond):
        pass


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_loss_runs_at_the_training_precision(monkeypatch, precision):
    """The loss calls train_forward, then its backward forward_train, both at the model's training precision when the loss was computed"""
    monkeypatch.setattr(_native, "require_cuda", lambda *t: None)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    monkeypatch.setattr(_native, "loss_noised_input", lambda x, noise, sigma, sd: x + noise * sigma.view(-1, 1, 1, 1))
    monkeypatch.setattr(_native, "denoiser_loss", lambda x, noise, sig, w, sd, f, kind: (f.flatten(1).mean(1), torch.ones_like(f)))
    cfg, inner, sd = model_of(CLASS)
    inner.load_state_dict(sd)
    log = []
    monkeypatch.setattr(type(inner), "engine", lambda self: _StubEngine(log))
    inner.set_train_precision(precision)
    model = K.config.make_denoiser_wrapper(cfg)(inner)
    x = torch.randn(2, 1, 16, 16)
    loss = model.loss(x, torch.randn_like(x), torch.tensor([0.5, 2.0]), class_cond=torch.tensor([1, 2]))
    inner.set_train_precision("fp32" if precision == "tf32" else "tf32")   # the backward keeps the forward's precision
    loss.sum().backward()
    calls = [c for c in log if c != "conditioning"]
    code = _native.PREC_TF32 if precision == "tf32" else _native.PREC_FP32
    assert calls == [("train_forward", 0.0, code), ("forward_train", code)]


def _inputs(B=2, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 1, 16, 16, generator=g) * 0.5
    noise = torch.randn(x.shape, generator=g)
    sigma = torch.exp(torch.randn(B, generator=g) * 1.2 - 0.4)
    return x, noise, sigma, {"class_cond": torch.tensor([3, 7][:B])}, torch.rand(B, generator=g) + 0.5


def test_restatement_rounds_exactly_the_token_stream_operands():
    """_Tf32Linear's forward, input gradient and weight gradient against the products of the rounded operands, and the mode replaces the
    token-stream Linears of the oracle's model only"""
    g = torch.Generator().manual_seed(1)
    a, w, d = (torch.randn(*s, generator=g, dtype=torch.float64) for s in ((3, 5, 24), (16, 24), (3, 5, 16)))
    a.requires_grad_()
    w.requires_grad_()
    with Tf32Linears([w]):
        y = a @ w.T
        z = a @ (w * 1).T   # not the weight itself: exact
    assert torch.equal(y, tf32_trunc(a.detach()) @ tf32_round(w.detach()).T)
    assert torch.equal(z, a.detach() @ w.detach().T)
    y.backward(d)
    assert torch.equal(a.grad, tf32_trunc(d) @ tf32_round(w.detach()))
    assert torch.equal(w.grad, tf32_trunc(d).reshape(-1, 16).T @ tf32_trunc(a.detach()).reshape(-1, 24))
    _, inner, _ = model_of(CLASS)
    keys = token_stream_keys(dict(inner.named_parameters()))
    assert len(keys) == 5 * 4 + 2 and "mapping.blocks.0.up_proj.weight" not in keys   # five attending layers, one merge, one split


def test_restatement_differs_measurably_from_fp32():
    """The tf32 restatement's gradients lie far from exact arithmetic compared with fp32 rounding, so the GPU tests can tell the routes apart"""
    cfg, _, sd = model_of(CLASS)
    x, noise, sigma, kw, gw = _inputs()
    l64, g64 = restated_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float64, False)
    l32, g32 = restated_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float32, False)
    t64, gt64 = restated_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float64, True)
    d_tf32 = sum(((gt64[k] - g64[k]).norm() / g64[k].norm()) ** 2 for k in g64 if g64[k].norm() > 0) ** 0.5
    d_fp32 = sum(((g32[k].double() - g64[k]).norm() / g64[k].norm()) ** 2 for k in g64 if g64[k].norm() > 0) ** 0.5
    assert d_tf32 > 1e-4 and d_tf32 > 20 * d_fp32, (d_tf32, d_fp32)
    assert (t64 - l64).abs().max() > 10 * (l32.double() - l64).abs().max()


LEVELS3 = {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [32, 32], "patch_size": [2, 2], "depths": [1, 1, 1],
                     "widths": [32, 48, 64], "d_ffs": [64, 96, 128], "mapping_width": 64, "mapping_depth": 1, "mapping_d_ff": 128,
                     "mapping_cond_dim": 12, "sigma_data": 0.5,
                     "self_attns": [{"type": "shifted-window", "d_head": 16, "window_size": 4}, {"type": "global", "d_head": 16},
                                    {"type": "none"}]}}


@pytest.mark.parametrize("spec", ["class", "levels3"])
def test_restatement_rewrites_every_token_stream_linear(spec):
    """The mode sees each token-stream weight of the oracle's model (restated_grads asserts it), on two levels with attention everywhere
    and on three levels whose last has none; the exact oracle's gradients of the other parameters are untouched"""
    cfg, _, sd = model_of(CLASS if spec == "class" else LEVELS3)
    g = torch.Generator().manual_seed(2)
    m = cfg["model"]
    x = torch.randn(1, m["input_channels"], *m["input_size"], generator=g) * 0.5
    noise, sigma = torch.randn(x.shape, generator=g), torch.tensor([0.8])
    kw = {"class_cond": torch.tensor([3])} if spec == "class" else {"aug_cond": torch.zeros(1, 9), "mapping_cond": torch.randn(1, 3, generator=g)}
    _, gt = restated_grads(cfg, sd, x, noise, sigma, kw, torch.ones(1), torch.float64, True)
    _, ge = restated_grads(cfg, sd, x, noise, sigma, kw, torch.ones(1), torch.float64, False)
    stream = token_stream_keys(gt)
    assert stream and all(not torch.equal(gt[k], ge[k]) for k in stream)


def test_wgrad_tf32_wrapper_refuses_mismatched_operands(monkeypatch):
    """The C entry point has no extents: the wrapper checks them before the call, so a mismatch raises instead of reading out of bounds"""
    monkeypatch.setattr(_native, "require_cuda", lambda *t: None)
    monkeypatch.setattr(_native, "lib", lambda: pytest.fail("reached the library"))
    dy, fine = torch.zeros(2 * 4 * 6, 40), torch.zeros(2, 8, 12, 24)
    for kwargs in ({"merge": (4, 5)}, {"merge": (3, 6)}, {"merge": (4, 6), "n_rows": 49}, {"merge": (0, 6)}):
        with pytest.raises(ValueError):
            _native.wgrad_tf32(dy, fine, **kwargs)
    with pytest.raises(ValueError):
        _native.wgrad_tf32(torch.zeros(3 * 4 * 6, 40), fine, merge=(4, 6))   # three images of gather rows, two of fine tokens
    with pytest.raises(ValueError):
        _native.wgrad_tf32(torch.zeros(10, 4), torch.zeros(9, 5))
    with pytest.raises(ValueError):
        _native.wgrad_tf32(torch.zeros(10, 4), torch.zeros(10, 5), out=torch.zeros(5, 4))
    with pytest.raises(ValueError):
        _native.wgrad_tf32(torch.zeros(10, 4), torch.zeros(10, 5), n_rows=11)
