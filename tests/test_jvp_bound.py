"""The tolerance of the GPU JVP tests (tests/test_gpu_jvp.py) separates the right derivative from near misses.

On the CPU oracle: torch.func.jvp (forward mode) and torch.autograd.functional.jvp (double backward, a different code path) agree within
the bound on three models that cover every attention kind; a forward-mode JVP with one derivative rule broken -- each installed over
the oracle function it belongs to, with the function's value unchanged -- falls outside it.
"""
import pytest
import torch

from conftest import load_fixture, synth_sd
from oracle import kdiff_oracle as O

NA3 = {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [64, 64], "patch_size": [4, 4],
                 "depths": [1, 1, 1], "widths": [128, 256, 512], "sigma_data": 0.5, "sigma_min": 1e-2, "sigma_max": 160,
                 "self_attns": [{"type": "neighborhood"}, {"type": "none"}, {"type": "global"}]}}


def check_tangent(got, want, what):
    """rel-L2 <= 1e-4 and elementwise |got - want| <= 1e-3 |want| + 1e-5 max|want| (the fp32 parity gate)"""
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    rel = float((got - want).norm() / want.norm())
    assert rel <= 1e-4, f"{what}: rel-L2 {rel:.3e}"
    err = (got - want).abs() - (1e-3 * want.abs() + 1e-5 * float(want.abs().max()))
    assert float(err.max()) <= 0, f"{what}: {int((err > 0).sum())} elements outside rtol 1e-3 / atol 1e-5 max|ref|"


def _model(name):
    import k_diffusion as K
    if name == "na3":
        cfg = K.config.load_config(NA3)
        shapes = {k: list(v.shape) for k, v in K.config.make_model(cfg).state_dict().items()}
    else:
        cfg, shapes, _ = load_fixture(name)
        cfg = K.config.load_config(cfg)
    mcfg = cfg["model"]
    om = O.make_denoiser(synth_sd(shapes, 1), mcfg)
    B = 2 if name == "cfg1_mnist" else 1
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, mcfg["input_channels"], *mcfg["input_size"], generator=g)
    v = torch.randint(0, 2, x.shape, generator=g).float() * 2 - 1
    sig = torch.tensor([0.7, 6.0][:B])
    kw = dict(class_cond=torch.tensor([1, 9])) if name == "cfg1_mnist" else {}
    return (lambda xx: om(xx, sig, **kw)), x, v


def _rms_no_mean(x, scale, eps=O.EPS):
    ms = torch.mean(x.float() ** 2, dim=-1, keepdim=True).detach()
    return x * (scale.float() * torch.rsqrt(ms + eps)).to(x.dtype)


def _cos_sim_no_projection(q, k, scale, eps=O.EPS):
    sq = torch.sqrt(scale)[:, None]
    q = q * (sq * torch.rsqrt(torch.sum(q ** 2, dim=-1, keepdim=True).detach() + eps))
    k = k * (sq * torch.rsqrt(torch.sum(k ** 2, dim=-1, keepdim=True).detach() + eps))
    return q, k


def _softmax_no_mean_subtraction(q, k, v, allow=None):
    logits = q @ k.transpose(-1, -2)
    if allow is not None:
        logits = logits.masked_fill(~allow, float("-inf"))
    p = torch.softmax(logits, dim=-1).detach()
    lt = logits if allow is None else logits.masked_fill(~allow, 0.0)
    return (p + p * (lt - lt.detach())) @ v                      # value P, tangent P dS instead of P (dS - sum P dS)


def _geglu_no_gelu_derivative(x, w):
    a, g = (x @ w.T).chunk(2, dim=-1)
    return a * torch.nn.functional.gelu(g.detach())


def _rope_not_on_tangent(x, theta, _orig=O.apply_rope):
    return _orig(x, theta).detach() + (x - x.detach())


def _denoiser_no_c_skip_tangent(inner, x, sigma, sigma_data, **kw):
    c_skip, c_out, c_in = [O._bcast(c, x.ndim) for c in O.karras_scalings(sigma, sigma_data)]
    return inner(x * c_in, sigma, **kw) * c_out + x.detach() * c_skip


NEAR_MISSES = {
    "rms_norm": _rms_no_mean,
    "cosine_sim_scale": _cos_sim_no_projection,
    "_softmax_av": _softmax_no_mean_subtraction,
    "linear_geglu": _geglu_no_gelu_derivative,
    "apply_rope": _rope_not_on_tangent,
    "denoiser_forward": _denoiser_no_c_skip_tangent,
}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["cfg1_mnist", "sw64", "na3"])
def test_bound_accepts_the_derivative_and_rejects_near_misses(name, monkeypatch):
    f, x, v = _model(name)
    y, jv = torch.func.jvp(f, (x,), (v,))
    y2, jv_rev = torch.autograd.functional.jvp(f, x, v)
    assert torch.equal(y, y2)
    check_tangent(jv_rev, jv, f"{name}: double-backward JVP")
    for fn, wrong in NEAR_MISSES.items():
        with monkeypatch.context() as mp:
            mp.setattr(O, fn, wrong)
            y_w, jv_w = torch.func.jvp(f, (x,), (v,))
        assert torch.allclose(y_w, y, rtol=1e-6, atol=1e-6 * float(y.abs().max())), f"{fn}: the near miss must keep the value"
        with pytest.raises(AssertionError):
            check_tangent(jv_w, jv, f"{name}: {fn}")
