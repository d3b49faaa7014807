"""The image_v1 U-Net engine (kdb_unet_*) on the H100: every stage against the fp32 oracle's restatement of that stage (fed the
engine's own input to it, computed in float64), the whole denoiser of the four reference configs against the reference's recorded
outputs and the oracle, samplers through the graph-captured executor, determinism, batch independence, the workspace check and
sample.py on a synthetic checkpoint."""
import json

import pytest
import torch
from torch.nn import functional as F

import k_diffusion as K
from conftest import GOLDEN, assert_close, load_npz
from oracle import kdiff_oracle as O
from oracle import unet_oracle as U
from oracle.fixtures import synth_sd

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
META = json.loads((GOLDEN / "unet_configs.json").read_text())
DEV = "cuda"


def build(name):
    cfg = K.config.load_config(META[name]["config"])
    sd = synth_sd(META[name]["shapes"], 1)
    model = K.config.make_model(cfg).eval().requires_grad_(False)
    model.load_state_dict(sd)
    model = model.to(DEV)
    return cfg, U.strip_prefix(sd), model, K.config.make_denoiser_wrapper(cfg)(model)


@pytest.mark.parametrize("name", sorted(META))
def test_forward_matches_reference_and_oracle(name):
    """B = 3, one sigma per image (sigma_min, 1, sigma_max), with and without a nonzero aug_cond"""
    cfg, sd, _, den = build(name)
    z = load_npz(f"unet_{name}.npz")
    x, sig, aug = z["x"].to(DEV), z["sigma"].to(DEV), z["aug_cond"].to(DEV)
    got, got_aug = den(x, sig), den(x, sig, aug_cond=aug)
    assert_close(got, z["denoised"], what=f"{name} vs reference")
    assert_close(got_aug, z["denoised_aug"], what=f"{name} aug_cond vs reference")
    want = U.make_denoiser(sd, cfg["model"])(z["x"], z["sigma"], aug_cond=z["aug_cond"])
    assert_close(got_aug, want, what=f"{name} aug_cond vs oracle")


def _stage_inputs(mcfg):
    """tap name -> (tap name of its input, oracle function of (input NCHW float64, cond float64), skip tap for the UBlock concat)"""
    depths, channels, attn, n = mcfg["depths"], mcfg["channels"], mcfg["self_attn_depths"], len(mcfg["depths"])
    stages, prev = {}, "patch_in"
    for i in range(n):
        if i > 0:
            stages[f"d{i}.down"] = (prev, lambda x, c: U.downsample(x), None)
            prev = f"d{i}.down"
        mods, _ = U.block_modules(depths[i], channels[max(0, i - 1)], channels[i], channels[i], attn[i], 1)
        for idx, kind, ci, cm, co in mods:
            stages[f"d{i}.{idx}"] = (prev, (kind, f"u_net.d_blocks.{i}.{idx}.", ci, cm, co), None)
            prev = f"d{i}.{idx}"
    skips = [f"d{i}.{U.block_modules(depths[i], 0, 0, 0, attn[i], 1)[1] - 1}" for i in range(n)]
    for k in range(n):
        i = n - 1 - k
        c_in = channels[i] * 2 if i < n - 1 else channels[i]
        mods, _ = U.block_modules(depths[i], c_in, channels[i], channels[max(0, i - 1)], attn[i], 0)
        for j, (idx, kind, ci, cm, co) in enumerate(mods):
            stages[f"u{i}.{idx}"] = (prev, (kind, f"u_net.u_blocks.{k}.{idx}.", ci, cm, co), skips[i] if (j == 0 and k > 0) else None)
            prev = f"u{i}.{idx}"
        if i > 0:
            stages[f"u{i}.up"] = (prev, lambda x, c: U.upsample(x), None)
            prev = f"u{i}.up"
    return stages


@pytest.mark.parametrize("name", ["mnist", "cifar10"])
def test_every_stage_against_the_oracle(name):
    """Each tap is checked against the oracle's restatement of its stage applied (in float64) to the engine's own tapped input, after
    the workspace was filled with NaN: conv3x3 at borders on 28/14/7 and 32/16/8 grids, the skip conv with c_in != c_out on the
    two-source concat, AdaGN, attention, down- and upsampling, patch-in."""
    cfg, sd, model, _ = build(name)
    mcfg = cfg["model"]
    unet = model.inner_model
    B, (H, W) = 2, mcfg["input_size"]
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, mcfg["input_channels"], H, W, generator=g).to(DEV)
    sig = torch.tensor([0.7, 9.0], device=DEV)
    aug = (torch.randn(B, 9, generator=g) * 0.5).to(DEV)
    eng = unet.engine(augment=True)
    cond = eng.conditioning(sig, aug)
    sd64 = {k: v.double() for k, v in sd.items()}
    cond_want = U.mapping(sd64, sig.cpu().double(), aug.cpu().double())
    assert_close(cond[:, -mcfg["mapping_out"]:], cond_want, rtol=1e-4, atol=1e-5, what="conditioning: mapping net")
    c64 = cond_want

    def run_tap(tap):
        need = eng.workspace_bytes(K._native.PREC_FP32, B, H, W)
        ws = eng._reserve(need, x.device)
        ws.view(torch.uint8)[: need - need % 4].view(torch.float32).fill_(float("nan"))
        buf = eng.arm_tap(tap, 1 << 24, x.device)
        eng.forward(x, sig, cond, eng.cond_stride, 0.0, K._native.PREC_FP32)
        n = eng.tap_count()
        assert n > 0, tap
        return buf[:n]

    def nchw(t, c):
        h = int(round((t.numel() / (B * c)) ** 0.5))
        return t.view(B, h, -1, c).permute(0, 3, 1, 2).cpu().double()

    stages = _stage_inputs(mcfg)
    got_pin = nchw(run_tap("patch_in"), mcfg["channels"][0])
    want_pin = F.conv2d(x.cpu().double(), sd64["proj_in.weight"], sd64["proj_in.bias"])
    assert_close(got_pin, want_pin, rtol=1e-4, atol=1e-5, what="patch_in")
    outs = {"patch_in": got_pin}
    for tap, (src, op, skip) in stages.items():
        inp = outs[src]
        if skip is not None:
            inp = torch.cat([inp, outs[skip]], dim=1)
        if isinstance(op, tuple):
            kind, p, ci, cm, co = op
            want = U.res_conv_block(sd64, p, inp, c64, ci, cm, co) if kind == "res" else U.self_attention(sd64, p, inp, c64)
            c_out = co
        else:
            want = op(inp, c64)
            c_out = inp.shape[1]
        got = nchw(run_tap(tap), c_out)
        assert torch.isfinite(got).all(), tap
        assert_close(got, want, rtol=1e-3, atol=1e-4, what=f"{name} stage {tap}")
        outs[tap] = got


def test_samplers_through_the_graph_executor_match_the_oracle():
    """Heun-10 against the reference's recorded trajectory; DPM++(2M) and Euler-ancestral with a BrownianTreeNoiseSampler (captured
    into a CUDA graph) against the oracle samplers fed the same noise"""
    cfg, sd, _, den = build("mnist")
    z = load_npz("unet_mnist.npz")
    S = K.sampling
    S.clear_graph_cache()
    n0 = len(S._graph_cache)
    got = S.sample_heun(den, z["heun_x"].to(DEV), z["heun_sigmas"].to(DEV), disable=True)
    assert len(S._graph_cache) == n0 + 1, "the sampler call was not captured"
    assert_close(got, z["heun"], what="heun-10 vs reference")
    oden = U.make_denoiser(sd, cfg["model"])
    x, sigmas = z["heun_x"], z["heun_sigmas"]
    assert_close(S.sample_dpmpp_2m(den, x.to(DEV), sigmas.to(DEV), disable=True), O.sample_dpmpp_2m(oden, x, sigmas), what="dpmpp_2m")
    xd = x.to(DEV)
    ns = S.BrownianTreeNoiseSampler(xd, float(sigmas[sigmas > 0].min()), float(sigmas.max()), seed=[3, 4])
    got = S.sample_euler_ancestral(den, xd, sigmas.to(DEV), disable=True, noise_sampler=ns)
    want = O.sample_euler_ancestral(oden, x, sigmas, noise_sampler=lambda s, t: ns(s, t).cpu())
    assert_close(got, want, what="euler_ancestral + Brownian tree")


def test_deterministic_and_batch_independent():
    _, _, model, den = build("cifar10")
    g = torch.Generator().manual_seed(9)
    x = (torch.randn(4, 3, 32, 32, generator=g) * 5).to(DEV)
    sig = torch.tensor([0.1, 1.0, 5.0, 40.0], device=DEV)
    aug = (torch.randn(4, 9, generator=g) * 0.5).to(DEV)
    a, b = den(x, sig, aug_cond=aug), den(x, sig, aug_cond=aug)
    assert torch.equal(a, b), "two calls differ"
    for i in range(4):
        alone = den(x[i:i + 1], sig[i:i + 1], aug_cond=aug[i:i + 1])
        assert torch.equal(alone, a[i:i + 1]), f"image {i} depends on its batch"


def test_workspace_too_short_and_bad_precision():
    _, _, model, _ = build("mnist")
    eng = model.inner_model.engine(augment=True)
    L = K._native.lib()
    x = torch.zeros(1, 1, 28, 28, device=DEV)
    sig = torch.ones(1, device=DEV)
    cond = eng.conditioning(sig)
    need = eng.workspace_bytes(K._native.PREC_FP32, 1, 28, 28)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    out = torch.empty_like(x)
    p = K._native.ptr
    args = lambda prec, nbytes: (eng._h, prec, 1, 28, 28, p(x), p(sig), 1.0, p(cond), 0, p(out), p(ws), nbytes, K._native.stream())
    assert L.kdb_unet_forward(*args(K._native.PREC_FP32, need // 2)) == -5
    assert L.kdb_unet_forward(*args(K._native.PREC_BF16, need)) == -2
    assert L.kdb_unet_workspace_bytes(eng._h, K._native.PREC_BF16, 1, 28, 28) == -2
    assert L.kdb_unet_forward(*args(K._native.PREC_FP32, need)) == 0
    torch.cuda.synchronize()


def test_log_likelihood_runs_on_forwards_only_and_derivatives_refuse():
    _, _, model, den = build("mnist")
    x = torch.randn(1, 1, 28, 28, generator=torch.Generator().manual_seed(2)).to(DEV) * 0.5
    ll, info = K.sampling.log_likelihood(den, x, 1e-2, 80.0, atol=1e-2, rtol=1e-2)
    assert torch.isfinite(ll).all()
    with pytest.raises(NotImplementedError):
        den.jvp(x, torch.ones(1, device=DEV), x)
    with pytest.raises(NotImplementedError):
        den(x.clone().requires_grad_(), torch.ones(1, device=DEV))


def test_sample_py_round_trip_on_a_synthetic_checkpoint(tmp_path, monkeypatch):
    import sys
    from safetensors.torch import save_file
    sys.path.insert(0, str(GOLDEN.parents[1] / "k-diffusion_b200"))
    import sample
    cfg = META["mnist"]["config"]
    ckpt = tmp_path / "mnist.safetensors"
    save_file({k: v.contiguous() for k, v in synth_sd(META["mnist"]["shapes"], 1).items()}, str(ckpt), metadata={"config": json.dumps(cfg)})
    monkeypatch.chdir(tmp_path)
    sample.main(["--checkpoint", str(ckpt), "-n", "3", "--batch-size", "2", "--steps", "4", "--prefix", "img", "--seed", "1"])
    files = sorted(p.name for p in tmp_path.glob("img_*.png"))
    assert files == ["img_00000.png", "img_00001.png", "img_00002.png"]
