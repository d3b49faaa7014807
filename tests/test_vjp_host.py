"""Host logic of the reverse-mode derivative without a GPU: torch.autograd through a native model makes one forward per evaluation and one
forward_vjp per backward, nothing changes with grad off, unsupported gradients raise, and Denoiser.vjp of a foreign model equals autograd.
The engine is replaced by a stub that evaluates the oracle on the CPU."""
import contextlib

import pytest
import torch

from conftest import synth_sd
from oracle import kdiff_oracle as O

import k_diffusion as K

TINY = {"model": {"type": "image_transformer_v2", "input_channels": 2, "input_size": [16, 16], "patch_size": [2, 2], "depths": [1, 1],
                  "widths": [32, 64], "mapping_cond_dim": 3, "sigma_data": 0.5,
                  "self_attns": [{"type": "shifted-window", "d_head": 16, "window_size": 4}, {"type": "global", "d_head": 16}]}}


class StubEngine:
    """Evaluates the oracle's inner model in place of the native engine, recording the entry points it is asked for."""
    cond_stride = 0

    def __init__(self, sd, mcfg):
        self.sd, self.mcfg, self.calls, self.mcond = sd, mcfg, [], None

    def _f(self, x, sig, sd):
        inner = lambda xx, s: O.model_forward(self.sd, self.mcfg, xx, s, mapping_cond=self.mcond)
        return O.denoiser_forward(inner, x, sig, sd) if sd > 0 else inner(x, sig)

    def check_class_range(self, class_cond):
        pass

    def conditioning(self, sig, aug, cc, mc):
        self.mcond = mc
        return torch.zeros(sig.shape[0], 1)

    def forward(self, x, sig, cond, stride, sd, precision, out=None):
        self.calls.append("forward")
        return self._f(x, sig, sd)

    def forward_vjp(self, x, u, sig, cond, stride, sd):
        self.calls.append("forward_vjp")
        f, pull = torch.func.vjp(lambda xx: self._f(xx, sig, sd), x)
        return f, pull(u)[0]


@pytest.fixture
def tiny(monkeypatch):
    from k_diffusion import _native
    monkeypatch.setattr(_native, "require_cuda", lambda *t: None)
    monkeypatch.setattr(_native, "f32c", lambda t: t.to(torch.float32).contiguous())
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    cfg = K.config.load_config(TINY)
    inner = K.config.make_model(cfg).eval()
    sd = synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, 1)
    inner.load_state_dict(sd)
    eng = StubEngine(sd, cfg["model"])
    inner.engine = lambda: eng
    model = K.config.make_denoiser_wrapper(cfg)(inner)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 2, 16, 16, generator=g)
    return model, eng, x, torch.tensor([0.7, 3.0]), torch.randn(2, 3, generator=g)


def test_autograd_makes_one_forward_and_one_forward_vjp_per_backward(tiny):
    model, eng, x, sig, mc = tiny
    u = torch.randn(x.shape, generator=torch.Generator().manual_seed(5))
    xg = x.clone().requires_grad_()
    d = model(xg, sig, mapping_cond=mc)
    assert d.grad_fn is not None and eng.calls == ["forward"]
    (g,) = torch.autograd.grad((d * u).sum(), xg)
    assert eng.calls == ["forward", "forward_vjp"]
    xr = x.clone().requires_grad_()
    want = O.denoiser_forward(lambda xx, s: O.model_forward(eng.sd, eng.mcfg, xx, s, mapping_cond=mc), xr, sig, 0.5)
    (g_want,) = torch.autograd.grad((want * u).sum(), xr)
    assert torch.allclose(d, want) and torch.allclose(g, g_want, rtol=1e-5, atol=1e-6)
    # a bf16 x gets a bf16 gradient
    xb = x.to(torch.bfloat16).requires_grad_()
    (gb,) = torch.autograd.grad((model(xb, sig, mapping_cond=mc).float() * u).sum(), xb)
    assert gb.dtype == torch.bfloat16


def test_nothing_changes_with_grad_off(tiny):
    model, eng, x, sig, mc = tiny
    with torch.no_grad():
        d = model(x.clone().requires_grad_(), sig, mapping_cond=mc)
    assert d.grad_fn is None
    d = model(x, sig, mapping_cond=mc)
    assert d.grad_fn is None and eng.calls == ["forward", "forward"]


def test_unsupported_gradients_raise(tiny):
    model, eng, x, sig, mc = tiny
    xg = x.clone().requires_grad_()
    with pytest.raises(RuntimeError, match="sigma"):
        model(xg, sig.clone().requires_grad_(), mapping_cond=mc)
    with pytest.raises(RuntimeError, match="mapping_cond"):
        model(xg, sig, mapping_cond=mc.clone().requires_grad_())
    with pytest.raises(RuntimeError, match="aug_cond"):
        model(xg, sig, mapping_cond=mc, aug_cond=torch.zeros(2, 9, requires_grad=True))
    with pytest.raises(RuntimeError, match="out="):
        model.inner_model.denoise(xg, sig, 0.5, mapping_cond=mc, out=torch.empty_like(x))
    assert eng.calls == []
    d = model(xg, sig, mapping_cond=mc)
    loss = d.square().sum()
    (g,) = torch.autograd.grad(loss, xg, create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(g.sum(), xg)                          # the backward is once_differentiable


def test_denoiser_vjp_foreign_model_equals_autograd(monkeypatch):
    from k_diffusion import _native
    monkeypatch.setattr(_native, "require_cuda", lambda *t: None)
    monkeypatch.setattr(_native, "f32c", lambda t: t.to(torch.float32).contiguous())

    def combine(f, x, sig, sd):
        c_skip, c_out, _ = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sig, sd)]
        return f * c_out + x * c_skip
    monkeypatch.setattr(_native, "precond_combine", combine)
    toy = lambda x, s, **kw: torch.tanh(x) * (1 + s[:, None, None, None]) + 0.3 * x.roll(1, -1) ** 2
    den = K.layers.Denoiser(toy, sigma_data=0.7)
    g = torch.Generator().manual_seed(2)
    x, u = torch.randn(3, 2, 5, 5, generator=g), torch.randn(3, 2, 5, 5, generator=g)
    sig = torch.tensor([0.2, 1.0, 9.0])
    d, gx = den.vjp(x, sig, u)
    xr = x.clone().requires_grad_()
    want = O.denoiser_forward(toy, xr, sig, 0.7)
    (g_want,) = torch.autograd.grad((want * u).sum(), xr)
    assert torch.allclose(d, want, rtol=1e-6, atol=1e-6) and torch.allclose(gx, g_want, rtol=1e-5, atol=1e-6)
