"""The external model wrappers (reference k_diffusion/external.py) without a GPU: oracle/external_oracle.py against the reference's
recorded outputs (tests/golden/external.npz, bit for bit), the wrappers' signatures, noise tables, sigma_to_t and scalings, and the
errors a CPU tensor or a training call meets."""
import inspect
import json

import pytest
import torch

import k_diffusion as K
from conftest import GOLDEN, assert_close, load_npz
from oracle import external_oracle as E
from oracle import kdiff_oracle as O

Z = load_npz("external.npz")
EXT = K.external


def _oracles():
    """name -> (oracle wrapper, x, kwargs): the wrappers oracle/make_golden_external.py recorded, around the same toy models"""
    ac = E.sd_alphas_cumprod()
    x4, x3, cond = Z["x4"], Z["x3"], Z["cond"]
    return {
        "compvis_q0": (E.CompVisDenoiserOracle(E.ToyCompVis(4), quantize=False), x4, dict(cond=cond)),
        "compvis_q1": (E.CompVisDenoiserOracle(E.ToyCompVis(4), quantize=True), x4, dict(cond=cond)),
        "compvis_fp16": (E.CompVisDenoiserOracle(E.ToyCompVis(4, out_dtype=torch.float16)), x4, dict(cond=cond)),
        "compvis_v": (E.CompVisVDenoiserOracle(E.ToyCompVis(4)), x4, dict(cond=cond, ignored=1)),
        "eps_ddpm": (E.DiscreteEpsDDPMDenoiserOracle(E.ToyModel(4), ac, quantize=True), x4, {}),
        "v_ddpm": (E.DiscreteVDDPMDenoiserOracle(E.ToyModel(4), ac, quantize=False), x4, {}),
        "openai": (E.OpenAIDenoiserOracle(E.ToyModel(3, learned_sigmas=True), E.ToyDiffusion()), x3, {}),
        "openai_nols": (E.OpenAIDenoiserOracle(E.ToyModel(3), E.ToyDiffusion(), quantize=True, has_learned_sigmas=False), x3, {}),
        "vdenoiser": (E.VDenoiserOracle(E.ToyModel(4, t_scale=1.0)), x4, {}),
    }


@pytest.mark.parametrize("name", sorted(_oracles()))
def test_oracle_forward_and_gradient_equal_the_reference_bit_for_bit(name):
    w, x, kw = _oracles()[name]
    sig = Z["sigma"]
    assert torch.equal(w(x, sig, **kw).detach(), Z[f"{name}_out"]), name
    xg = x.clone().requires_grad_()
    grad = torch.autograd.grad((w(xg, sig, **kw) * Z["loss_w"][:, :x.shape[1]]).sum(), xg)[0]
    assert torch.equal(grad, Z[f"{name}_grad_x"]), name


@pytest.mark.parametrize("kind", ["eps", "v"])
@pytest.mark.parametrize("sampler", ["euler", "heun", "dpmpp_2m", "lms", "euler_ancestral"])
def test_oracle_sampler_trajectories_match_the_reference(kind, sampler):
    inner = E.ToyCompVis(4)
    w = E.CompVisDenoiserOracle(inner) if kind == "eps" else E.CompVisVDenoiserOracle(inner)
    x, sigmas, ea = Z[f"{kind}_traj_x"], Z[f"{kind}_traj_sigmas"], dict(cond=Z[f"{kind}_traj_cond"])
    assert torch.equal(w.get_sigmas(8), sigmas)
    if sampler == "euler_ancestral":
        it = iter(Z[f"{kind}_traj_noise"])
        got = O.sample_euler_ancestral(w, x, sigmas, ea, noise_sampler=lambda a, b: next(it))
    else:
        got = getattr(O, f"sample_{sampler}")(w, x, sigmas, ea)
    assert_close(got, Z[f"{kind}_traj_{sampler}"], rtol=1e-5, atol=1e-5, what=f"{kind} {sampler}")


def test_signatures_equal_the_reference():
    want = json.loads((GOLDEN / "external_signatures.json").read_text())
    assert len(want) >= 35
    for label, sig in want.items():
        _, cls, method = label.split(".")
        got = [[n, p.kind.name, None if p.default is inspect._empty else repr(p.default)]
               for n, p in inspect.signature(getattr(getattr(EXT, cls), method)).parameters.items()]
        assert got == sig, label
    for cls in ("VDenoiser", "DiscreteEpsDDPMDenoiser", "OpenAIDenoiser", "CompVisDenoiser", "DiscreteVDDPMDenoiser", "CompVisVDenoiser"):
        assert f"external.{cls}.forward" in want and issubclass(getattr(EXT, cls), torch.nn.Module)


@pytest.mark.parametrize("quantize", [False, True])
def test_tables_and_sigma_to_t_equal_the_reference(quantize):
    """sigma_to_t stays the inherited torch op sequence: the int64 indices and the interpolated t are the reference's exactly"""
    w = EXT.CompVisDenoiser(E.ToyCompVis(4), quantize=quantize)
    assert torch.equal(w.sigmas, Z["sigmas"]) and torch.equal(w.log_sigmas, Z["log_sigmas"])
    assert torch.equal(w.get_sigmas(12), Z["get_sigmas_12"])
    q = Z[f"cv_q{int(quantize)}_query"]
    t = w.sigma_to_t(q)
    want = Z[f"cv_q{int(quantize)}_t"]
    assert t.dtype == want.dtype == (torch.int64 if quantize else torch.float32)
    assert torch.equal(t, want)
    assert set(w.state_dict()) == {"sigmas", "log_sigmas"} | {f"inner_model.{k}" for k in E.ToyCompVis(4).state_dict()}


def test_openai_and_vdenoiser_schedules_equal_the_reference():
    oa = EXT.OpenAIDenoiser(E.ToyModel(3, learned_sigmas=True), E.ToyDiffusion())
    assert oa.sigmas.dtype == torch.float32 and torch.equal(oa.sigmas, Z["openai_sigmas"])
    assert oa.has_learned_sigmas and not oa.quantize and oa.sigma_data == 1.0
    v = EXT.VDenoiser(E.ToyModel(4))
    assert torch.equal(v.sigma_to_t(Z["vdenoiser_query"]), Z["vdenoiser_t"])
    assert torch.equal(v.t_to_sigma(torch.tensor([0.0, 0.1, 0.5, 0.9, 0.999])), Z["vdenoiser_t_to_sigma"])


def test_get_scalings_equal_the_oracle():
    sig = torch.tensor([0.0, 0.03, 1.0, 14.6, 157.0])
    for w in (EXT.VDenoiser(None), EXT.DiscreteVDDPMDenoiser(None, E.sd_alphas_cumprod(), False)):
        for a, b in zip(w.get_scalings(sig), E.v_scalings(sig, 1.0)):
            assert torch.equal(a, b)
    w = EXT.DiscreteEpsDDPMDenoiser(None, E.sd_alphas_cumprod(), False)
    for a, b in zip(w.get_scalings(sig), E.eps_scalings(sig, 1.0)):
        assert torch.equal(a, b)


def test_cpu_tensors_and_training_raise():
    x, sig = Z["x4"], Z["sigma"]
    for w in (EXT.CompVisDenoiser(E.ToyCompVis(4)), EXT.CompVisVDenoiser(E.ToyCompVis(4)), EXT.VDenoiser(E.ToyModel(4)),
              EXT.OpenAIDenoiser(E.ToyModel(4, learned_sigmas=True), E.ToyDiffusion())):
        with pytest.raises(RuntimeError, match="CUDA tensors only"):
            w(x, sig, cond=Z["cond"]) if "CompVis" in type(w).__name__ else w(x, sig)
        with pytest.raises(NotImplementedError):
            w.loss(x, torch.randn_like(x), sig)
