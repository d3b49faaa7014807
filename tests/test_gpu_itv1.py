"""image_transformer_v1 on the H100, through the transformer engine (KdbModelConfig.family = image_transformer_v1): the fp32 path
against the reference's recorded outputs and the oracle on the three configs of oracle/make_golden_itv1.py, the bf16 path within
twice the reference's own bf16 distance, the `.qkv` tap against the oracle's QKNorm + RoPE in the engine's column order, the
tensor-core route of the bf16 forward, the derivatives against torch.func of the oracle, CUDA-graph replay against eager launches,
and sample.py on a synthetic checkpoint."""
import json
import math

import pytest
import torch
from torch.nn.attention import SDPBackend, sdpa_kernel

import k_diffusion as K
from conftest import GOLDEN, assert_close, load_npz
from oracle import itv1_oracle as V
from oracle import kdiff_oracle as O
from oracle.fixtures import synth_sd

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
META = json.loads((GOLDEN / "itv1_meta.json").read_text())["configs"]
NAMES = sorted(META)
DEV = "cuda"


def build(name, precision="fp32"):
    cfg = K.config.load_config(META[name]["config"])
    sd = synth_sd(META[name]["shapes"], 1)
    model = K.config.make_model(cfg).eval().requires_grad_(False)
    model.load_state_dict(sd)
    model = model.to(DEV).set_precision(precision)
    return cfg, sd, model, K.config.make_denoiser_wrapper(cfg)(model)


def cond_kw(z, dev=DEV):
    return {"class_cond": z["class_cond"].to(dev)} if "class_cond" in z else {}


def assert_as_close_as_the_reference(got, ref32, want64, what):
    """got against the float64 oracle at the fp32 tolerance, with atol raised to twice the largest distance of the reference's own fp32
    result from the float64 oracle where that is larger: the synthetic QKNorm scales reach the clamp (softmax temperature 100), which
    amplifies fp32 rounding beyond 1e-5 in the reference itself"""
    atol = max(1e-5, 2 * float((ref32.double() - want64.double()).abs().max()))
    assert_close(got, want64, atol=atol, what=what)


def rel_l2(a, b):
    return float((a.detach().cpu().double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("name", NAMES)
def test_fp32_matches_oracle_and_reference(name):
    """B = 3, one sigma per image (sigma_min, 1, sigma_max), with and without aug_cond, per-sample class rows, and the raw inner model,
    against the float64 oracle (assert_as_close_as_the_reference)"""
    cfg, sd, model, den = build(name)
    z = load_npz(f"itv1_{name}.npz")
    x, sig, aug = z["x"].to(DEV), z["sigma"].to(DEV), z["aug_cond"].to(DEV)
    kw, kw_cpu = cond_kw(z), cond_kw(z, "cpu")
    sd64 = {k: v.double() for k, v in sd.items()}
    x64, s64 = z["x"].double(), z["sigma"].double()
    oden = V.make_denoiser(sd64, cfg["model"])
    cases = [("denoised", den(x, sig, **kw), oden(x64, s64, **kw_cpu)),
             ("denoised_aug", den(x, sig, aug_cond=aug, **kw), oden(x64, s64, aug_cond=z["aug_cond"].double(), **kw_cpu)),
             ("inner", model(x, sig, **kw), V.model_forward(sd64, cfg["model"], x64, s64, **kw_cpu))]
    for key, got, want in cases:
        assert_as_close_as_the_reference(got, z[key], want, what=f"{name} {key}")


@pytest.mark.parametrize("name", NAMES)
def test_bf16_forward_within_the_reference_bf16_budget(name):
    _, _, _, den = build(name, "bf16")
    z = load_npz(f"itv1_{name}.npz")
    got = den(z["x"].to(DEV), z["sigma"].to(DEV), **cond_kw(z))
    budget = META[name]["bf16_budget"]["forward_rel_l2"]
    assert torch.isfinite(got).all()
    assert rel_l2(got, z["denoised"]) < 2 * budget, f"{name}: rel_l2 {rel_l2(got, z['denoised']):.3e} vs 2 x {budget:.3e}"


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_heun10(precision):
    """the graph-captured sampler on the MNIST-sized class-conditional config against the reference's trajectory"""
    cfg, sd, _, den = build("mnist", precision)
    z = load_npz("itv1_mnist.npz")
    S = K.sampling
    S.clear_graph_cache()
    got = S.sample_heun(den, z["heun_x"].to(DEV), z["heun_sigmas"].to(DEV), extra_args=dict(class_cond=z["heun_class_cond"].to(DEV)),
                        disable=True)
    assert len(S._graph_cache) == 1, "the sampler call was not captured"
    if precision == "fp32":
        sd64 = {k: v.double() for k, v in sd.items()}
        want = O.sample_heun(V.make_denoiser(sd64, cfg["model"]), z["heun_x"].double(), z["heun_sigmas"].double(),
                             dict(class_cond=z["heun_class_cond"]))
        # normwise, against a tenth of the reference's own bf16 distance: over ten steps the clamped temperatures (softmax scale 100)
        # amplify fp32 rounding, in the reference as here (its fp32 trajectory is 3.4e-4 from the float64 one, relative L2; this
        # engine's was 7.8e-4 on an H100)
        assert rel_l2(got, want) <= 0.1 * META["mnist"]["bf16_budget"]["heun10_rel_l2"], rel_l2(got, want)
    else:
        budget = META["mnist"]["bf16_budget"]["heun10_rel_l2"]
        assert rel_l2(got, z["heun"]) < 2 * budget


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_graph_replay_equals_eager(precision, monkeypatch):
    _, _, _, den = build("cifar", precision)
    g = torch.Generator().manual_seed(9)
    x = (torch.randn(2, 3, 32, 32, generator=g) * 160).to(DEV)
    sigmas = K.sampling.get_sigmas_karras(6, 1e-2, 160, device=DEV)
    K.sampling.clear_graph_cache()
    graph = K.sampling.sample_heun(den, x, sigmas, disable=True)
    assert len(K.sampling._graph_cache) == 1
    monkeypatch.setenv("KDB200_CUDA_GRAPH", "0")
    eager = K.sampling.sample_heun(den, x, sigmas, disable=True)
    assert torch.equal(graph, eager)


def oracle_qk(sd, mcfg, x, sigma, class_cond):
    """the oracle's q and k of block 0 after QKNorm + RoPE, [B, T, nh, e] each, in float64"""
    ph, pw = mcfg["patch_size"]
    B, c, H, W = x.shape
    h, w = H // ph, W // pw
    t = x.view(B, c, h, ph, w, pw).permute(0, 2, 4, 1, 3, 5).reshape(B, h * w, c * ph * pw) @ sd["in_proj.weight"].T
    emb = O.fourier_features((torch.log(sigma) / 4)[..., None], sd["time_emb.weight"]) @ sd["time_in_proj.weight"].T
    emb = emb + O.fourier_features(t.new_zeros(B, 9), sd["aug_emb.weight"]) @ sd["aug_in_proj.weight"].T
    if class_cond is not None:
        emb = emb + sd["class_emb.weight"][class_cond]
    cond = O.mapping_network(sd, emb)
    p = "blocks.0.self_attn."
    xn = O.rms_norm(t, (cond @ sd[p + "norm.linear.weight"].T)[:, None, :] + 1)
    nh = t.shape[-1] // V.D_HEAD
    q, k, _ = (xn @ sd[p + "qkv_proj.weight"].T).view(B, h * w, 3, nh, V.D_HEAD).permute(2, 0, 3, 1, 4).unbind(0)
    theta = V.rope_theta(V.make_axial_pos(h, w, ph / pw, dtype=x.dtype), sd[p + "pos_emb.freqs_h"], sd[p + "pos_emb.freqs_w"])
    rot = lambda u: V.apply_rope(V.qk_norm(u, sd[p + "qk_norm.scale"]), theta).transpose(1, 2)
    return rot(q), rot(k)


@pytest.mark.parametrize("name", NAMES)
def test_qkv_tap_is_the_oracle_qk_in_engine_column_order(name):
    cfg, sd, model, _ = build(name)
    z = load_npz(f"itv1_{name}.npz")
    x, sig = z["x"].to(DEV), z["sigma"].to(DEV)
    kw = cond_kw(z)
    eng = model.engine()
    cond = model.conditioning(sig, None, kw.get("class_cond"))
    B, T, C = x.shape[0], cfg["model"]["input_size"][0] * cfg["model"]["input_size"][1] // math.prod(cfg["model"]["patch_size"]), cfg["model"]["width"]
    buf = eng.arm_tap("layer0.qkv", B * T * 3 * C, DEV)
    eng.forward(x.contiguous(), sig, cond, eng.cond_stride, 0.0, K._native.PREC_FP32)
    torch.cuda.synchronize()
    assert eng.tap_count() == B * T * 3 * C
    got = buf.cpu().view(B, T, 3, C // V.D_HEAD, V.D_HEAD)
    sd64 = {k: v.double() for k, v in sd.items()}
    q, k = oracle_qk(sd64, cfg["model"], z["x"].double(), z["sigma"].double(), z.get("class_cond"))
    perm = V.head_permutation()
    s = V.D_HEAD ** -0.25              # the engine's q, k carry the square root of SDPA's 1 / sqrt(d_head) each
    assert_close(got[:, :, 0], q[..., perm] * s, what=f"{name} q")
    assert_close(got[:, :, 1], k[..., perm] * s, what=f"{name} k")


def test_bf16_cifar_forward_runs_on_the_tensor_core_kernels():
    _, _, model, den = build("cifar", "bf16")
    g = torch.Generator().manual_seed(3)
    x = torch.randn(8, 3, 32, 32, generator=g).to(DEV)
    sig = torch.full((8,), 2.0, device=DEV)
    den(x, sig)                                     # positions and tables of this grid
    torch.cuda.synchronize()
    before = K._native.launch_breakdown()
    den(x, sig)
    torch.cuda.synchronize()
    after = K._native.launch_breakdown()
    d = {k: after[k] - before.get(k, 0) for k in after}
    assert d["gemm_tc"] >= 8 * 4 and d["attn_tc"] >= 8, d
    for fam in ("gemm_simt", "attn_generic", "qknorm_rope", "geglu"):
        assert d.get(fam, 0) == 0, (fam, d)


def test_derivatives_match_torch_func_of_the_oracle():
    cfg, sd, model, den = build("edge")
    mcfg = cfg["model"]
    sd64 = {k: v.double() for k, v in sd.items()}
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 3, 24, 40, generator=g, dtype=torch.float64) * 2
    v = torch.randn(2, 3, 24, 40, generator=g, dtype=torch.float64)
    u = torch.randn(2, 3, 24, 40, generator=g, dtype=torch.float64)
    sig = torch.tensor([0.7, 3.0], dtype=torch.float64)
    f = lambda xi: V.model_forward(sd64, mcfg, xi, sig)
    with sdpa_kernel(SDPBackend.MATH):              # the CPU flash kernel of scaled_dot_product_attention has no forward-mode AD
        want_f, want_t = torch.func.jvp(f, (x,), (v,))
        _, vjp_fn = torch.func.vjp(f, x)
        (want_g,) = vjp_fn(u)
    xd, sd_ = x.float().to(DEV), sig.float().to(DEV)
    got_f, got_t = model.jvp(xd, sd_, v.float().to(DEV))
    assert_close(got_f, want_f, what="jvp primal")
    assert_close(got_t, want_t, what="jvp tangent")
    got_f2, got_g = model.vjp(xd, sd_, u.float().to(DEV))
    assert_close(got_f2, want_f, what="vjp primal")
    assert_close(got_g, want_g, what="vjp gradient")
    xg = xd.clone().requires_grad_(True)
    with torch.enable_grad():
        model(xg, sd_).backward(u.float().to(DEV))
    assert_close(xg.grad, want_g, what="torch.autograd gradient")


def test_sample_py_round_trip_on_a_synthetic_checkpoint(tmp_path, monkeypatch):
    import sys
    from safetensors.torch import save_file
    sys.path.insert(0, str(GOLDEN.parents[1] / "k-diffusion_b200"))
    import sample
    cfg = META["cifar"]["config"]
    ckpt = tmp_path / "itv1.safetensors"
    save_file({k: v.contiguous() for k, v in synth_sd(META["cifar"]["shapes"], 1).items()}, str(ckpt), metadata={"config": json.dumps(cfg)})
    monkeypatch.chdir(tmp_path)
    sample.main(["--checkpoint", str(ckpt), "-n", "3", "--batch-size", "2", "--steps", "4", "--prefix", "img", "--seed", "1",
                 "--precision", "bf16"])
    assert sorted(p.name for p in tmp_path.glob("img_*.png")) == ["img_00000.png", "img_00001.png", "img_00002.png"]
