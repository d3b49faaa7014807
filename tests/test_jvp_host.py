"""Host logic of log_likelihood(jvp=True) without a GPU: a native Denoiser gets exactly one forward-mode engine call per right-hand side
(the engine is replaced by a stub evaluator that computes the oracle's torch.func.jvp), foreign models keep autograd."""
import numpy as np
import torch

from conftest import load_fixture, synth_sd
from oracle import kdiff_oracle as O

import k_diffusion as K

S = K.sampling


def _ll_fn():
    fn = S.log_likelihood
    while hasattr(fn, "__wrapped__"):
        fn = fn.__wrapped__                           # below the device guard (no CUDA here)
    return fn


def _stub_natives(monkeypatch):
    from k_diffusion import _native
    monkeypatch.setattr(_native, "require_cuda", lambda *t: None)
    monkeypatch.setattr(_native, "f32c", lambda t: t.to(torch.float32).contiguous())
    monkeypatch.setattr(_native, "lincomb", lambda ts, cs, out=None: sum(np.float32(c) * t for t, c in zip(ts, cs)))
    monkeypatch.setattr(_native, "rk_error", lambda err, y0, y1, atol, rtol:
                        float((err / (atol + rtol * torch.maximum(y0.abs(), y1.abs()))).pow(2).mean().sqrt()))


def test_log_likelihood_jvp_routes_native_denoiser_to_one_forward_jvp(monkeypatch):
    _stub_natives(monkeypatch)
    cfg, shapes, _ = load_fixture("cfg1_mnist")
    omodel = O.make_denoiser(synth_sd(shapes, 1), cfg["model"])
    den = K.config.make_denoiser_wrapper(cfg)(K.config.make_model(cfg))
    assert den.is_native()
    calls = []

    class StubEvaluator:                              # stands in for the engine
        def __init__(self, model, x, extra_args, sigmas):
            self.sig, self.ea = sigmas, extra_args

        def __call__(self, k, x):
            calls.append(("forward", self.sig[k]))
            raise AssertionError("the JVP route must not run plain forwards")

        def jvp(self, k, x, v):
            calls.append(("jvp", self.sig[k]))
            return torch.func.jvp(lambda xx: omodel(xx, torch.full((x.shape[0],), self.sig[k]), **self.ea), (x,), (v,))

    monkeypatch.setattr(S, "_Evaluator", StubEvaluator)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 1, 28, 28, generator=g) * 0.4 + 0.1
    v = torch.randint(0, 2, x.shape, generator=g).float() * 2 - 1
    ea = {"class_cond": torch.tensor([1, 9])}
    rhs, count = S._likelihood_rhs(den, x, ea, v, 1e-2, jvp=True)
    for i, sigma in enumerate((0.02, 0.7, 30.0)):
        xs = x * (1 + sigma)
        with torch.no_grad():
            d, d_ll = rhs(sigma, (xs, torch.zeros(2)))
        assert calls[-1] == ("jvp", sigma) and len(calls) == i + 1 and count[0] == i + 1
        with torch.enable_grad():
            xg = xs.clone().requires_grad_()
            dd = (xg - omodel(xg, torch.full((2,), sigma), **ea)) / sigma
            want = (v * torch.autograd.grad((dd * v).sum(), xg)[0]).flatten(1).sum(1)
        assert float((d_ll - want).abs().max()) <= 1e-4 * float(want.abs().max()), (sigma, d_ll, want)
    calls.clear()
    with torch.no_grad():
        ll, info = _ll_fn()(den, x, 1e-2, 80., extra_args=ea, v=v, jvp=True)
    assert len(calls) == info["fevals"] and all(c[0] == "jvp" for c in calls)
    ll_o, _ = O.log_likelihood(omodel, x, 1e-2, 80., extra_args=ea, v=v)
    assert float((ll - ll_o).abs().max()) <= 1e-3 * float(ll_o.abs().max())


def test_log_likelihood_jvp_keeps_autograd_for_foreign_models(monkeypatch):
    _stub_natives(monkeypatch)
    toy = lambda x, s, **kw: x / (1 + s[:, None, None, None] ** 2) + 0.1 * torch.tanh(x)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 1, 4, 4, generator=g)
    v = torch.randint(0, 2, x.shape, generator=g).float() * 2 - 1
    with torch.no_grad():
        a, ia = _ll_fn()(toy, x, 1e-2, 80., v=v)
        b, ib = _ll_fn()(toy, x, 1e-2, 80., v=v, jvp=True)
    assert torch.equal(a, b) and ia == ib
