"""GPU parity tests: the CUDA path (through the C ABI via k_diffusion) against the CPU oracle on
the same seeded inputs and against the reference-generated golden fixtures.

Tolerance for the fp32 exact path is the north-star gate rtol 1e-3 / atol 1e-5; integer / schedule
paths are bit-exact (tests/test_host_logic.py).  bf16 tolerances are stated where used.
"""
import json

import pytest
import torch

import k_diffusion as K
from conftest import GOLDEN, assert_close, load_fixture, load_npz, synth_sd
from oracle import kdiff_oracle as O

pytestmark = pytest.mark.gpu
S = K.sampling
DEV = "cuda"


def build(stem_or_cfg, seed=1, precision="fp32"):
    if isinstance(stem_or_cfg, str):
        cfg, shapes, z = load_fixture(stem_or_cfg)
    else:
        cfg, shapes, z = K.config.load_config(stem_or_cfg), None, None
    inner = K.config.make_model(cfg)
    if shapes is None:
        shapes = {k: list(v.shape) for k, v in inner.state_dict().items()}
    sd = synth_sd(shapes, seed)
    inner.load_state_dict(sd)
    inner = inner.to(DEV).eval().set_precision(precision)
    model = K.config.make_denoiser_wrapper(cfg)(inner)
    return cfg, sd, inner, model, z


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


# ------------------------------------------------------------------------------------------
# solver kernels
# ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 3, 4, 1023, 4096 + 5, 3 * 256 * 256 * 2])
def test_solver_kernels_match_formulas(n):
    from k_diffusion import _native as N
    g = torch.Generator(device=DEV).manual_seed(n)
    x, d1, x2, d2, nz = (torch.randn(n, device=DEV, generator=g) for _ in range(5))
    assert_close(N.euler_step(x, d1, -0.37), x + (x - d1) * -0.37, rtol=1e-6, atol=1e-6)
    assert_close(N.euler_step(x, d1, -0.37, noise=nz, cn=0.8), x + (x - d1) * -0.37 + nz * 0.8, rtol=1e-6, atol=1e-6)
    assert_close(N.heun_correct(x, d1, x2, d2, -0.2, -1.3), x + ((x - d1) * -0.2 + (x2 - d2) * -1.3), rtol=1e-6, atol=1e-6)
    assert_close(N.dpmpp_2m_step(x, d1, d2, 0.7, -0.3, 1.4, -0.4), 0.7 * x + 0.3 * (1.4 * d1 - 0.4 * d2), rtol=1e-6, atol=1e-6)
    assert_close(N.dpmpp_2m_step(x, d1, None, 0.7, -0.3, 1.0, 0.0), 0.7 * x + 0.3 * d1, rtol=1e-6, atol=1e-6)
    assert_close(N.lincomb([x, d1, x2, d2, nz], [1, 2, -3, 0.5, 4]), x + 2 * d1 - 3 * x2 + 0.5 * d2 + 4 * nz, rtol=1e-5, atol=1e-5)
    # unaligned views take the scalar path; in-place aliasing is allowed
    if n > 8:
        xv, dv = x[1:], d1[1:]
        assert_close(N.euler_step(xv, dv, 0.25), xv + (xv - dv) * 0.25, rtol=1e-6, atol=1e-6)
    y = x.clone()
    N.euler_step(y, d1, 0.5, out=y)
    assert_close(y, x + (x - d1) * 0.5, rtol=1e-6, atol=1e-6)


def test_precond_and_to_d():
    from k_diffusion import _native as N
    g = torch.Generator(device=DEV).manual_seed(0)
    x, f = torch.randn(5, 3, 8, 8, device=DEV, generator=g), torch.randn(5, 3, 8, 8, device=DEV, generator=g)
    sigma = torch.tensor([0.01, 0.5, 3.0, 80.0, 160.0], device=DEV)
    cs, co, ci = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sigma, 0.5)]
    assert_close(N.precond_scale_in(x, sigma, 0.5), x * ci, rtol=1e-6, atol=1e-7)
    assert_close(N.precond_combine(f, x, sigma, 0.5), f * co + x * cs, rtol=1e-6, atol=1e-7)
    assert_close(S.to_d(x, sigma, f), (x - f) / sigma.view(-1, 1, 1, 1), rtol=1e-6, atol=1e-7)
    assert_close(S.to_d(x, torch.tensor(2.0, device=DEV), f), (x - f) / 2.0, rtol=1e-6, atol=1e-7)


# ------------------------------------------------------------------------------------------
# model forward, fp32 exact path
# ------------------------------------------------------------------------------------------

def test_cfg1_mnist_forward_vs_golden_and_oracle():
    cfg, sd, inner, model, z = build("cfg1_mnist")
    x, cc, sig = z["x"].to(DEV), z["class_cond"].to(DEV), z["sigma"].to(DEV)
    assert_close(inner(x * 0.01, sig, class_cond=cc), z["inner"], what="inner vs golden")
    assert_close(inner(x * 0.01, sig, aug_cond=z["aug_cond"].to(DEV), class_cond=cc), z["inner_aug"], what="inner_aug vs golden")
    assert_close(model(x, sig, class_cond=cc), z["denoised"], what="denoised vs golden")
    # fresh inputs against the live oracle
    g = torch.Generator().manual_seed(99)
    x2 = torch.randn(3, 1, 28, 28, generator=g) * 5
    s2, c2 = torch.tensor([0.02, 1.7, 33.0]), torch.tensor([10, 3, 7])
    want = O.make_denoiser(sd, cfg["model"])(x2, s2, class_cond=c2)
    assert_close(model(x2.to(DEV), s2.to(DEV), class_cond=c2.to(DEV)), want, what="denoised vs oracle")
    with pytest.raises(ValueError, match="class_cond"):
        model(x, sig)


def test_layer_taps_vs_oracle_cfg1():
    """Intermediate activations of the first layer against the oracle (localises any divergence)."""
    cfg, sd, inner, model, z = build("cfg1_mnist")
    x, cc, sig = z["x"][:2].to(DEV) * 0.01, z["class_cond"][:2].to(DEV), z["sigma"][:2].to(DEV)
    eng = inner.engine()
    buf = eng.arm_tap("patch_in", 2 * 49 * 256, DEV)
    inner(x, sig, class_cond=cc)
    assert eng.tap_count() == 2 * 49 * 256
    want = O.token_merge(x.cpu().movedim(-3, -1), sd["patch_in.proj.weight"], 4, 4)
    assert_close(buf.view(2, 7, 7, 256), want, what="patch_in")


def test_sw64_forward_and_taps():
    cfg, sd, inner, model, z = build("sw64")
    x, sig = z["x"].to(DEV), z["sigma"].to(DEV)
    assert_close(inner(x * 0.01, sig), z["inner"], what="inner vs golden")
    assert_close(model(x, sig), z["denoised"], what="denoised vs golden")


def test_cfg2_sw256_forward_b1():
    cfg, sd, inner, model, z = build("cfg2_sw256")
    g = torch.Generator().manual_seed(int(z["seed"]))
    x = (torch.randn(1, 3, 256, 256, generator=g) * 160).to(DEV)
    sig = z["sigma"].to(DEV)
    o = inner(x * 0.01, sig)
    assert_close(o[..., ::4, ::4], z["inner_sub"], what="inner_sub")
    assert_close(model(x, sig)[..., ::4, ::4], z["denoised_sub"], what="denoised_sub")


NA_CFG = {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [64, 64], "patch_size": [4, 4],
                    "depths": [2, 2, 2], "widths": [128, 256, 512], "sigma_data": 0.5, "sigma_min": 1e-2, "sigma_max": 160}}


def test_neighborhood_model_vs_oracle():
    """7x7 neighbourhood attention (default self_attns).  natten is absent from the reference tree, so the
    oracle's masked-attention restatement is the bar here (parity vs real NATTEN unpinned)."""
    cfg, sd, inner, model, _ = build(NA_CFG)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 3, 64, 64, generator=g) * 20
    sig = torch.tensor([0.7, 25.0])
    assert_close(model(x.to(DEV), sig.to(DEV)), O.make_denoiser(sd, cfg["model"])(x, sig), what="NA denoised")


def test_neighborhood_model_bf16_tensor_core_path():
    """128x128 input -> 32x32 tokens at level 0: the tensor-core neighbourhood kernel (level 1 = 16x16 stays on the generic one)."""
    raw = {"model": dict(NA_CFG["model"], input_size=[128, 128], depths=[1, 1, 1])}
    cfg, sd, inner, model, _ = build(raw, precision="bf16")
    g = torch.Generator().manual_seed(8)
    x = torch.randn(2, 3, 128, 128, generator=g) * 10
    sig = torch.tensor([0.9, 12.0])
    want = O.make_denoiser(sd, cfg["model"])(x, sig)
    assert rel_l2(model(x.to(DEV), sig.to(DEV)), want) < 2e-2


def test_cfg5_shape_512_forward_b1():
    """BASELINE configs[4] model (512x512, widths 256/512/1024, depths 2/2/4, NA,NA,global) at B=1: bf16 path vs the fp32 oracle.
    Exercises the 1024-token global attention (8 key blocks, two-pass) and the NA kernel on 128x128 / 64x64 token grids."""
    raw = {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [512, 512], "patch_size": [4, 4],
                     "depths": [2, 2, 4], "widths": [256, 512, 1024], "sigma_data": 0.5, "sigma_min": 1e-2, "sigma_max": 160}}
    cfg, sd, inner, model, _ = build(raw, precision="bf16")
    g = torch.Generator().manual_seed(9)
    x = torch.randn(1, 3, 512, 512, generator=g) * 5
    sig = torch.tensor([2.0])
    want = O.make_denoiser(sd, cfg["model"])(x, sig)
    got = model(x.to(DEV), sig.to(DEV))
    assert torch.isfinite(got).all() and rel_l2(got, want) < 2e-2


def test_nonsquare_and_mapping_cond():
    raw = {"model": {"type": "image_transformer_v2", "input_channels": 2, "input_size": [32, 64], "patch_size": [2, 4],
                     "depths": [1, 2], "widths": [64, 128], "mapping_cond_dim": 5, "sigma_data": 1.0,
                     "self_attns": [{"type": "shifted-window", "d_head": 32, "window_size": 4}, {"type": "global", "d_head": 64}]},
           "dataset": {"type": "x", "num_classes": 3}}
    cfg, sd, inner, model, _ = build(raw)
    g = torch.Generator().manual_seed(6)
    x = torch.randn(3, 2, 32, 64, generator=g)
    sig = torch.tensor([0.3, 2.0, 9.0])
    kw = dict(class_cond=torch.tensor([0, 3, 1]), mapping_cond=torch.randn(3, 5, generator=g), aug_cond=torch.randn(3, 9, generator=g))
    want = O.make_denoiser(sd, cfg["model"])(x, sig, **kw)
    got = model(x.to(DEV), sig.to(DEV), **{k: v.to(DEV) for k, v in kw.items()})
    assert_close(got, want, what="nonsquare")


# ------------------------------------------------------------------------------------------
# samplers
# ------------------------------------------------------------------------------------------

def test_cfg1_samplers_vs_golden():
    """BASELINE.json configs[0]: sample_heun 10 steps, MNIST transformer, batch 4, fp32 parity gate."""
    cfg, sd, inner, model, z = build("cfg1_mnist")
    x, sigmas = z["x"].to(DEV), z["sigmas"].to(DEV)
    ea = dict(class_cond=z["class_cond"].to(DEV))
    assert_close(S.sample_heun(model, x, sigmas, extra_args=ea, disable=True), z["heun"], what="heun")
    assert_close(S.sample_dpmpp_2m(model, x, sigmas, extra_args=ea, disable=True), z["dpmpp_2m"], what="dpmpp_2m")
    assert_close(S.sample_euler(model, x, sigmas, extra_args=ea, disable=True), z["euler"], what="euler")
    it = iter(z["noise"].to(DEV))
    got = S.sample_euler_ancestral(model, x, sigmas, extra_args=ea, disable=True, noise_sampler=lambda a, b: next(it))
    assert_close(got, z["euler_ancestral"], what="euler_ancestral")


def test_sw64_samplers_graph_and_eager(monkeypatch):
    cfg, sd, inner, model, z = build("sw64")
    x, sigmas = z["x"].to(DEV), z["sigmas"].to(DEV)
    S.clear_graph_cache()
    g1 = S.sample_heun(model, x, sigmas, disable=True)                 # captured + replayed
    g2 = S.sample_heun(model, x, sigmas, disable=True)                 # replay from cache
    assert_close(g1, z["heun"], what="heun (graph)")
    assert torch.equal(g1, g2)
    monkeypatch.setenv("KDB200_CUDA_GRAPH", "0")
    e1 = S.sample_heun(model, x, sigmas, disable=True)
    assert torch.equal(e1, g1), "graph replay must be bit-identical to eager launches"
    assert_close(S.sample_dpmpp_2m(model, x, sigmas, disable=True), z["dpmpp_2m"], what="dpmpp_2m")
    seen = []
    S.sample_heun(model, x, sigmas, disable=True, callback=lambda d: seen.append((d["i"], float(d["sigma"]), tuple(d["denoised"].shape))))
    assert [s[0] for s in seen] == list(range(6)) and seen[0][2] == tuple(x.shape)


def test_opaque_model_samplers_vs_golden():
    """Arbitrary callables keep working: fused solver kernels around an opaque model(x, sigma)."""
    z = load_npz("toy_samplers.npz")
    toy2 = lambda x, s, **kw: x / (1 + s[:, None, None, None] ** 2) + 0.1 * torch.tanh(x)
    x, sigmas = z["x"].to(DEV), z["sigmas"].to(DEV)
    for name in ("sample_euler", "sample_heun", "sample_dpmpp_2m"):
        assert_close(getattr(S, name)(toy2, x, sigmas, disable=True), z[name], rtol=1e-4, atol=1e-5, what=name)
    it = iter(z["noise"].to(DEV))
    assert_close(S.sample_euler_ancestral(toy2, x, sigmas, disable=True, noise_sampler=lambda a, b: next(it)), z["sample_euler_ancestral"],
                 rtol=1e-4, atol=1e-5)
    it = iter(z["noise"].to(DEV))
    assert_close(S.sample_euler_ancestral(toy2, x, sigmas, disable=True, eta=0.5, s_noise=0.9, noise_sampler=lambda a, b: next(it)),
                 z["sample_euler_ancestral_eta05"], rtol=1e-4, atol=1e-5)
    # Denoiser around an opaque inner model uses the two preconditioning kernels
    inner = lambda xi, s, **kw: 0.3 * xi
    den = K.Denoiser(inner, sigma_data=0.5)
    sig = torch.tensor([0.5, 2.0, 9.0], device=DEV)
    want = O.denoiser_forward(lambda xi, s: 0.3 * xi, z["x"], sig.cpu(), 0.5)
    assert_close(den(x, sig), want, rtol=1e-5, atol=1e-6)
    # x is not modified in place and dtype/device are preserved
    x0 = x.clone()
    out = S.sample_heun(toy2, x, sigmas, disable=True)
    assert torch.equal(x, x0) and out.dtype == x.dtype and out.device == x.device


@pytest.mark.parametrize("name,fn,kw", [("euler_churn20", "sample_euler", dict(s_churn=20.)),
                                        ("heun_churn3_window", "sample_heun", dict(s_churn=3., s_tmin=0.1, s_tmax=30., s_noise=1.1)),
                                        ("dpm_2_churn2", "sample_dpm_2", dict(s_churn=2.))])
def test_churn_vs_reference_with_replayed_draws(name, fn, kw, monkeypatch):
    """s_churn > 0 against the reference (oracle/make_golden_churn.py).  Noise is only drawn on steps with gamma > 0 (quirk Q1), so the
    reference's recorded draws of exactly those steps are replayed."""
    z = load_npz("toy_churn.npz")
    toy2 = lambda x, s, **k: x / (1 + s[:, None, None, None] ** 2) + 0.1 * torch.tanh(x)
    n = len(z["sigmas"]) - 1
    gamma = lambda s_: min(kw["s_churn"] / n, 2 ** 0.5 - 1) if kw.get("s_tmin", 0.) <= float(s_) <= kw.get("s_tmax", float("inf")) else 0.
    it = iter([z[name + "_eps"][i].to(DEV) for i in range(n) if gamma(z["sigmas"][i]) > 0])
    monkeypatch.setattr(torch, "randn_like", lambda t, *a, **k: next(it))
    got = getattr(S, fn)(toy2, z["x"].to(DEV), z["sigmas"].to(DEV), disable=True, **kw)
    assert_close(got, z[name], rtol=1e-4, atol=2e-5, what=name)
    assert next(it, None) is None


def test_churn_matches_statistics():
    toy = lambda x, s, **kw: 0.5 * x
    x = torch.ones(4, 1, 64, 64, device=DEV)
    sig = S.get_sigmas_karras(8, 1e-2, 80, device=DEV)
    torch.manual_seed(0)
    a = S.sample_heun(toy, x, sig, disable=True, s_churn=20.0)
    torch.manual_seed(0)
    b = S.sample_heun(toy, x, sig, disable=True, s_churn=20.0)
    assert torch.equal(a, b) and float(a.std()) > 0                      # stochastic, reproducible under manual_seed
    c = S.sample_heun(toy, x, sig, disable=True)
    assert float(c.std()) == 0.0


# ------------------------------------------------------------------------------------------
# size-independent properties at the BASELINE sizes (256x256, batch 32)
# ------------------------------------------------------------------------------------------

def test_batch_independence_256():
    """Each image depends only on its own latent: row b of a B=8 batch == the same image run alone."""
    cfg, sd, inner, model, _ = build("cfg2_sw256")
    x = K.parallel.init_noise(K.parallel.sample_seeds(1, 0, 8), (3, 256, 256), 160.0, DEV)
    sig = torch.full([8], 3.0, device=DEV)
    full = model(x, sig)
    solo = model(x[5:6].contiguous(), sig[:1])
    assert_close(full[5:6], solo, rtol=1e-4, atol=1e-5, what="batch independence")
    assert torch.isfinite(full).all()


@pytest.mark.parametrize("sampler,steps", [("sample_heun", 4), ("sample_dpmpp_2m", 5)])
def test_shard_invariance_256_b32(sampler, steps):
    """B=32 at 256x256 (cfg2 shape): sampling a shard of the batch gives the same images as the full batch."""
    cfg, sd, inner, model, _ = build("cfg2_sw256", precision="bf16")
    seeds = K.parallel.sample_seeds(3, 0, 32)
    x = K.parallel.init_noise(seeds, (3, 256, 256), 160.0, DEV)
    x_shard = K.parallel.init_noise(seeds[8:16], (3, 256, 256), 160.0, DEV)
    assert torch.equal(x[8:16], x_shard)
    sigmas = S.get_sigmas_karras(steps, 1e-2, 160, device=DEV)
    full = getattr(S, sampler)(model, x, sigmas, disable=True)
    part = getattr(S, sampler)(model, x_shard, sigmas, disable=True)
    assert torch.isfinite(full).all() and float(full.abs().max()) < 50
    assert rel_l2(full[8:16], part) < 1e-5


# ------------------------------------------------------------------------------------------
# bf16 path: tolerance vs the fp32 oracle (the reference's bf16 mode is autocast, SURVEY 8d)
# ------------------------------------------------------------------------------------------

def test_bf16_forward_close_to_fp32_oracle():
    cfg, sd, inner, model, z = build("sw64", precision="bf16")
    x, sig = z["x"].to(DEV), z["sigma"].to(DEV)
    got = model(x, sig)
    # bf16 token stream (8-bit mantissa) through 24 residual blocks: relative L2 error budget 2e-2
    assert rel_l2(got, z["denoised"]) < 2e-2
    g1 = S.sample_heun(model, x, z["sigmas"].to(DEV), disable=True)
    assert rel_l2(g1, z["heun"]) < 5e-2


def test_autocast_selects_bf16():
    cfg, sd, inner, model, z = build("sw64", precision="auto")
    from k_diffusion import _native
    assert inner.resolved_precision() == _native.PREC_FP32
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert inner.resolved_precision() == _native.PREC_BF16


# ------------------------------------------------------------------------------------------
# noise
# ------------------------------------------------------------------------------------------

def test_philox_noise_properties():
    like = torch.empty(6, 3, 64, 64, device=DEV)
    seeds = K.parallel.sample_seeds(11, 0, 6)
    smp = S.PhiloxNoiseSampler(like, seeds)
    a, b = smp(1.0, 0.5), smp(0.5, 0.2)
    assert abs(float(a.mean())) < 0.02 and abs(float(a.std()) - 1) < 0.02 and abs(float((a * b).mean())) < 0.02
    again = S.PhiloxNoiseSampler(like[:2], seeds[2:4])
    assert torch.equal(again(1.0, 0.5), a[2:4])                           # shard invariance
    k = float(((a - a.mean()) ** 4).mean() / a.var() ** 2)
    assert abs(k - 3.0) < 0.1                                             # normal kurtosis


def test_brownian_tree_properties():
    like = torch.empty(4, 3, 128, 128, device=DEV)
    seeds = [5, 6, 7, 8]
    tree = S.BatchedBrownianTree(like, 0.01, 160.0, seed=seeds)
    w_ac, w_ab, w_bc = tree(2.0, 40.0), tree(2.0, 11.0), tree(11.0, 40.0)
    assert_close(w_ab + w_bc, w_ac, rtol=1e-4, atol=1e-4, what="additivity")
    assert abs(float(w_ac.var()) / 38.0 - 1) < 0.03                        # Var[W(b)-W(a)] = |b-a|
    assert abs(float(tree(0.02, 0.05).var()) / 0.03 - 1) < 0.03
    assert torch.equal(tree(40.0, 2.0), -w_ac)                            # sign handling (sampling.py:82-88)
    assert torch.equal(S.BatchedBrownianTree(like[:2], 0.01, 160.0, seed=seeds[1:3])(2.0, 40.0), w_ac[1:3])
    assert abs(float((w_ab * w_bc).mean())) / (9 * 29) ** 0.5 < 0.02      # independent increments
    ns = S.BrownianTreeNoiseSampler(like, 0.01, 160.0, seed=seeds)
    n1 = ns(torch.tensor(40.0), torch.tensor(2.0))
    assert abs(float(n1.std()) - 1) < 0.02 and torch.equal(n1, ns(40.0, 2.0))
    single = S.BatchedBrownianTree(like, 0.01, 160.0, seed=3)
    assert single(1.0, 2.0).shape == like.shape and not single.batched
    flipped = S.BatchedBrownianTree(like, 160.0, 0.01, seed=seeds)
    assert torch.equal(flipped(2.0, 40.0), -w_ac)


def test_euler_ancestral_brownian_shard_invariant():
    """cfg4 shape of work at reduced batch: Euler-ancestral + Brownian tree, per-sample seeds."""
    cfg, sd, inner, model, _ = build(NA_CFG, precision="bf16")
    seeds = K.parallel.sample_seeds(9, 0, 6)
    x = K.parallel.init_noise(seeds, (3, 64, 64), 160.0, DEV)
    sigmas = S.get_sigmas_karras(6, 1e-2, 160, device=DEV)
    run = lambda xs, sd_: S.sample_euler_ancestral(model, xs, sigmas, disable=True, noise_sampler=S.BrownianTreeNoiseSampler(xs, 1e-2, 160, seed=sd_))
    full, part = run(x, seeds), run(x[2:5].contiguous(), seeds[2:5])
    assert torch.isfinite(full).all() and rel_l2(full[2:5], part) < 1e-5


def test_launch_counter_and_loaded_library():
    from k_diffusion import _native
    before = _native.launch_count()
    x = torch.ones(8, device=DEV)
    _native.euler_step(x, x, 0.5)
    assert _native.launch_count() == before + 1
    assert "libkdb200.so" in open("/proc/self/maps").read()
