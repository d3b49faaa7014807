"""The external model wrappers (reference k_diffusion/external.py) on the GPU: each forward against oracle/external_oracle.py run by
torch on the same GPU (bit for bit, including the t the inner model receives), against the reference's CPU outputs, gradients, jvp,
sampler trajectories, log_likelihood, launch count and CUDA-graph capture."""
import pytest
import torch

import k_diffusion as K
from conftest import assert_close, load_npz
from k_diffusion import _native
from oracle import external_oracle as E
from oracle import kdiff_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
EXT = K.external


def _z():
    return {k: (v.to(DEV) if v.is_floating_point() else v) for k, v in load_npz("external.npz").items()}


def _pair(name):
    """(native wrapper, oracle wrapper, inner toy model, x, kwargs) sharing one toy model on the GPU"""
    z = _z()
    ac = E.sd_alphas_cumprod().to(DEV)
    x4, x3, kw_c = z["x4"], z["x3"], dict(cond=z["cond"])
    table = {
        "compvis_q0": (EXT.CompVisDenoiser, E.CompVisDenoiserOracle, lambda: E.ToyCompVis(4), dict(quantize=False), x4, kw_c),
        "compvis_q1": (EXT.CompVisDenoiser, E.CompVisDenoiserOracle, lambda: E.ToyCompVis(4), dict(quantize=True), x4, kw_c),
        "compvis_fp16": (EXT.CompVisDenoiser, E.CompVisDenoiserOracle, lambda: E.ToyCompVis(4, out_dtype=torch.float16), {}, x4, kw_c),
        "compvis_v": (EXT.CompVisVDenoiser, E.CompVisVDenoiserOracle, lambda: E.ToyCompVis(4), {}, x4, dict(kw_c, ignored=1)),
        "eps_ddpm": (lambda m, **k: EXT.DiscreteEpsDDPMDenoiser(m, ac, **k), lambda m, **k: E.DiscreteEpsDDPMDenoiserOracle(m, ac, **k),
                     lambda: E.ToyModel(4), dict(quantize=True), x4, {}),
        "v_ddpm": (lambda m, **k: EXT.DiscreteVDDPMDenoiser(m, ac, **k), lambda m, **k: E.DiscreteVDDPMDenoiserOracle(m, ac, **k),
                   lambda: E.ToyModel(4), dict(quantize=False), x4, {}),
        "openai": (lambda m, **k: EXT.OpenAIDenoiser(m, E.ToyDiffusion(), device=DEV), lambda m, **k: E.OpenAIDenoiserOracle(m, E.ToyDiffusion(), device=DEV),
                   lambda: E.ToyModel(3, learned_sigmas=True), {}, x3, {}),
        "openai_nols": (lambda m, **k: EXT.OpenAIDenoiser(m, E.ToyDiffusion(), quantize=True, has_learned_sigmas=False, device=DEV),
                        lambda m, **k: E.OpenAIDenoiserOracle(m, E.ToyDiffusion(), quantize=True, has_learned_sigmas=False, device=DEV),
                        lambda: E.ToyModel(3), {}, x3, {}),
        "vdenoiser": (EXT.VDenoiser, E.VDenoiserOracle, lambda: E.ToyModel(4, t_scale=1.0), {}, x4, {}),
    }
    ours, oracle, make_inner, ckw, x, kw = table[name]
    inner = make_inner().to(DEV)
    w = ours(inner, **ckw).to(DEV)
    return w, oracle(inner, **ckw), inner, x, kw


NAMES = ["compvis_q0", "compvis_q1", "compvis_fp16", "compvis_v", "eps_ddpm", "v_ddpm", "openai", "openai_nols", "vdenoiser"]


def _toy(inner):
    return inner.model if isinstance(inner, E.ToyCompVis) else inner


@pytest.mark.parametrize("name", NAMES)
def test_forward_equals_the_oracle_on_the_gpu_bit_for_bit(name):
    w, o, inner, x, kw = _pair(name)
    seen = []
    h = _toy(inner).register_forward_pre_hook(lambda mod, args: seen.append((args[0].clone(), args[1].clone())))
    try:
        with torch.no_grad():
            got, want = w(x, _z()["sigma"], **kw), o(x, _z()["sigma"], **kw)
    finally:
        h.remove()
    (xa, ta), (xb, tb) = seen
    assert ta.dtype == tb.dtype and torch.equal(ta, tb), "t the inner model receives"
    assert torch.equal(xa, xb), "c_in x the inner model receives"
    assert got.dtype == want.dtype == torch.float32 and torch.equal(got, want)
    # the toy model's tanh / sin differ from the CPU's by an ulp, which c_out (up to 14.6 here) scales: rtol 1e-6 of the output's scale
    ref = _z()[f"{name}_out"]
    assert_close(got, ref, rtol=1e-6, atol=1e-6 * float(ref.abs().max()), what=f"{name} vs the reference's CPU output")


@pytest.mark.parametrize("name", NAMES)
def test_gradients_match_oracle_autograd(name):
    w, o, inner, x, kw = _pair(name)
    sig, lw = _z()["sigma"], _z()["loss_w"][:, :x.shape[1]]
    param = _toy(inner).weight
    grads, outs = [], []
    for model in (w, o):
        xg = x.clone().requires_grad_()
        outs.append(model(xg, sig, **kw))
        grads.append(torch.autograd.grad((outs[-1] * lw).sum(), (xg, param)))
    assert torch.equal(outs[0], outs[1]), "forward through the autograd Functions"
    (gx, gp), (ox, op) = grads
    assert_close(gx, ox, rtol=1e-6, atol=1e-7, what=f"{name} grad x")
    assert_close(gp, op, rtol=1e-6, atol=1e-6, what=f"{name} grad of the inner weight")
    ref = _z()[f"{name}_grad_x"]
    assert_close(ox, ref, rtol=1e-5, atol=1e-5 * float(ref.abs().max()), what=f"{name} grad x vs the reference's CPU gradient")


@pytest.mark.parametrize("name", ["compvis_q0", "compvis_fp16", "compvis_v", "openai", "vdenoiser"])
def test_jvp_matches_the_oracle(name):
    w, o, inner, x, kw = _pair(name)
    sig = _z()["sigma"]
    t = torch.randn(x.shape, generator=torch.Generator().manual_seed(9)).to(DEV)
    fa, ja = torch.func.jvp(lambda xx: w(xx, sig, **kw), (x,), (t,))
    fb, jb = torch.func.jvp(lambda xx: o(xx, sig, **kw), (x,), (t,))
    assert torch.equal(fa, fb)
    assert_close(ja, jb, rtol=1e-6, atol=1e-7, what=f"{name} torch.func.jvp")
    import torch.autograd.forward_ad as fwAD
    with fwAD.dual_level():
        jc = fwAD.unpack_dual(w(fwAD.make_dual(x, t), sig, **kw)).tangent
    assert_close(jc, jb, rtol=1e-6, atol=1e-7, what=f"{name} forward_ad")


def test_sigma_that_requires_grad_raises():
    w, _, _, x, kw = _pair("compvis_q0")
    with pytest.raises(RuntimeError, match="not sigma"):
        w(x, _z()["sigma"].clone().requires_grad_(), **kw)


@pytest.mark.parametrize("kind", ["eps", "v"])
@pytest.mark.parametrize("sampler", ["euler", "heun", "dpmpp_2m", "lms", "euler_ancestral"])
def test_sampler_trajectories_match_the_reference(kind, sampler):
    z = _z()
    inner = E.ToyCompVis(4).to(DEV)
    w = (EXT.CompVisDenoiser(inner) if kind == "eps" else EXT.CompVisVDenoiser(inner)).to(DEV)
    x, sigmas, ea = z[f"{kind}_traj_x"], z[f"{kind}_traj_sigmas"], dict(cond=z[f"{kind}_traj_cond"])
    kw = {}
    if sampler == "euler_ancestral":
        it = iter(z[f"{kind}_traj_noise"])
        kw = dict(noise_sampler=lambda a, b: next(it))
    got = getattr(K.sampling, f"sample_{sampler}")(w, x, sigmas, extra_args=ea, disable=True, **kw)
    assert_close(got, z[f"{kind}_traj_{sampler}"], what=f"{kind} {sampler}")


def test_log_likelihood_through_a_wrapper_matches_the_oracle():
    g = torch.Generator().manual_seed(21)
    x = torch.randn(2, 4, 8, 8, generator=g) * 0.5
    v = torch.randint(0, 2, x.shape, generator=g).float() * 2 - 1
    cond = torch.randn(2, 4, 8, 8, generator=g)
    w = EXT.CompVisDenoiser(E.ToyCompVis(4).to(DEV)).to(DEV)
    ll, info = K.sampling.log_likelihood(w, x.to(DEV), 0.03, 14.0, extra_args=dict(cond=cond.to(DEV)), v=v.to(DEV))
    ll_o, info_o = O.log_likelihood(E.CompVisDenoiserOracle(E.ToyCompVis(4)), x, 0.03, 14.0, extra_args=dict(cond=cond), v=v)
    # two correct dopri5 integrations at the default tolerances differ by a few rtol * |ll| (the step sequence decides)
    assert float((ll.cpu() - ll_o).abs().max()) <= 1e-3 * float(ll_o.abs().max()), (ll, ll_o)
    assert abs(info["fevals"] - info_o["fevals"]) <= 18


@pytest.mark.parametrize("name", ["compvis_q1", "openai", "vdenoiser"])
def test_one_call_is_two_launches(name):
    """in the samplers' no_grad loop (plain calls) and with autograd recording (through the autograd Functions)"""
    w, _, _, x, kw = _pair(name)
    sig = _z()["sigma"]
    for mode in (torch.no_grad, torch.enable_grad):
        with mode():
            w(x, sig, **kw)
            n0 = _native.launch_count()
            w(x, sig, **kw)
            assert _native.launch_count() - n0 == 2, mode


@pytest.mark.parametrize("name", ["compvis_q1", "compvis_v", "vdenoiser"])
def test_one_evaluation_captures_in_a_cuda_graph(name):
    """No host sync inside a wrapper call: around a capture-safe toy model it records into a graph whose replay equals eager."""
    w, _, _, x, kw = _pair(name)
    sig = _z()["sigma"].clone()
    xs = x.clone()
    with torch.no_grad():
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            w(xs, sig, **kw)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = w(xs, sig, **kw)
        for scale in (1.0, -0.5):
            xs.copy_(x * scale)
            sig.copy_(_z()["sigma"] * (2 - scale))
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, w(xs, sig, **kw)), scale


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("shape", [(3, 4, 8, 8), (2, 3, 5, 5), (1, 6, 4, 4)])
def test_kernels_equal_torch_for_every_dtype_layout_and_dropped_term(dtype, shape):
    """kdb_external_combine / scale_in on the vectorised and the scalar path, a strided channel slice of the model output, and with
    x or f dropped (the derivative forms), against the reference's torch expressions on the same GPU"""
    g = torch.Generator().manual_seed(sum(shape))
    B = shape[0]
    x = (torch.randn(shape, generator=g) * 20).to(DEV)
    full = (torch.randn(B, 2 * shape[1], *shape[2:], generator=g) * 3).to(DEV, dtype)
    sigma = torch.tensor([0.0, 1e-4, 0.7, 14.6, 1e4][:B] if B > 1 else [3.3]).to(DEV)
    f = full[:, :shape[1]]                                              # a view with its own batch stride
    col = lambda t: t[:, None, None, None]
    c_skip, c_out, c_in = (col(c) for c in E.v_scalings(sigma, 1.0))
    assert torch.equal(_native.external_scale_in(x, sigma), x * c_in)
    assert torch.equal(_native.external_combine(_native.EXTERNAL_EPS, f, x, sigma), x + f * col(-sigma))
    assert torch.equal(_native.external_combine(_native.EXTERNAL_V, f, x, sigma), f * c_out + x * c_skip)
    assert torch.equal(_native.external_combine(_native.EXTERNAL_EPS, f, None, sigma), f * col(-sigma))
    assert torch.equal(_native.external_combine(_native.EXTERNAL_V, f, None, sigma), f * c_out)
    assert torch.equal(_native.external_combine(_native.EXTERNAL_V, None, x, sigma), x * c_skip)
    assert torch.equal(_native.external_combine(_native.EXTERNAL_EPS, f.contiguous(), x, sigma), x + f * col(-sigma))
