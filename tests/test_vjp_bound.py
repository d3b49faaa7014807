"""The tolerance of the GPU VJP tests (tests/test_gpu_vjp.py) separates the right reverse-mode derivative from near misses.

On the CPU oracle: torch.func.vjp agrees within check_tangent with u^T J assembled from the full forward-mode Jacobian (vmap of jvp over
the input basis, an independent code path); a reverse-mode derivative with one rule broken -- each installed over the oracle function
it belongs to, with the function's value unchanged -- falls outside the bound on three models that cover every attention kind.
"""
import pytest
import torch

from conftest import load_fixture, synth_sd
from oracle import kdiff_oracle as O
from test_jvp_bound import NEAR_MISSES, _model, check_tangent


def _lerp_no_skip_gradient(start, end, weight, _orig=torch.lerp):
    """TokenSplit's lerp with the gradient of the skip connection dropped"""
    return _orig(start.detach(), end, weight)


def _vjp(f, x, u):
    y, pull = torch.func.vjp(f, x)
    return y, pull(u)[0]


@pytest.mark.timeout(900)
def test_vjp_matches_the_transposed_forward_mode_jacobian():
    """cfg1, one image: u^T J from the 784 columns J e_i of torch.func.jvp (vmapped over the basis) against torch.func.vjp"""
    cfg, shapes, _ = load_fixture("cfg1_mnist")
    import k_diffusion as K
    mcfg = K.config.load_config(cfg)["model"]
    om = O.make_denoiser(synth_sd(shapes, 1), mcfg)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(1, 1, 28, 28, generator=g)
    u = torch.randn(1, 1, 28, 28, generator=g)
    sig, cc = torch.tensor([1.7]), torch.tensor([4])
    f = lambda xx: om(xx, sig, class_cond=cc)
    _, want = _vjp(f, x, u)
    basis = torch.eye(x.numel()).view(-1, *x.shape)
    cols = torch.func.vmap(lambda e: torch.func.jvp(f, (x,), (e,))[1], chunk_size=98)(basis)   # [784, 1, 1, 28, 28]: J e_i
    got = (cols.flatten(1) @ u.flatten()).view_as(x)
    check_tangent(got, want, "cfg1: u^T J from the forward-mode Jacobian")


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["cfg1_mnist", "sw64", "na3"])
def test_bound_rejects_reverse_mode_near_misses(name, monkeypatch):
    f, x, _ = _model(name)
    u = torch.randn(x.shape, generator=torch.Generator().manual_seed(9))
    y, gx = _vjp(f, x, u)
    misses = [(O, fn, wrong) for fn, wrong in NEAR_MISSES.items()]
    if name != "cfg1_mnist":                                      # cfg1 has one level, so no TokenSplit
        misses.append((torch, "lerp", _lerp_no_skip_gradient))
    for mod, fn, wrong in misses:
        with monkeypatch.context() as mp:
            mp.setattr(mod, fn, wrong)
            y_w, g_w = _vjp(f, x, u)
        assert torch.allclose(y_w, y, rtol=1e-6, atol=1e-6 * float(y.abs().max())), f"{fn}: the near miss must keep the value"
        with pytest.raises(AssertionError):
            check_tangent(g_w, gx, f"{name}: {fn}")
