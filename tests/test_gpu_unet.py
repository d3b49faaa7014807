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


def build(name, meta=META):
    cfg = K.config.load_config(meta[name]["config"])
    sd = synth_sd(meta[name]["shapes"], 1)
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


def unet_engine(model, mcfg):
    """the native engine of a make_model result, with the conditioning its config's wrapper forms"""
    augment = mcfg["augment_wrapper"]
    return (model.inner_model if augment else model).engine(augment=augment)


def oracle_mapping_cond(mcfg, B, aug=None, mc=None):
    """the mapping_cond the bare model sees (augmentation.py:97-104): [aug_cond or zeros(9), mapping_cond] with the wrapper"""
    if not mcfg["augment_wrapper"]:
        return mc
    a = torch.zeros(B, 9, dtype=torch.float64) if aug is None else aug
    return a if mc is None else torch.cat([a, mc], dim=1)


def check_every_stage(name, cfg, sd, model, x, sig, aug=None, mc=None):
    """Each tap against the oracle's restatement of its stage applied (in float64) to the engine's own tapped input, after the workspace
    was filled with NaN; every tap holds exactly B * h * w * C floats, with (h, w) the grid of its level."""
    mcfg = cfg["model"]
    eng = unet_engine(model, mcfg)
    B, _, H, W = x.shape
    cond = eng.conditioning(sig, aug, mapping_cond=mc)
    sd64 = {k: v.double() for k, v in sd.items()}
    c64 = U.mapping(sd64, sig.cpu().double(), oracle_mapping_cond(mcfg, B, *(None if t is None else t.cpu().double() for t in (aug, mc))))
    assert_close(cond[:, -mcfg["mapping_out"]:], c64, rtol=1e-4, atol=1e-5, what=f"{name} conditioning: mapping net")

    def run_tap(tap, level, c):
        need = eng.workspace_bytes(K._native.PREC_FP32, B, H, W)
        ws = eng._reserve(need, x.device)
        ws.view(torch.uint8)[: need - need % 4].view(torch.float32).fill_(float("nan"))
        buf = eng.arm_tap(tap, 1 << 24, x.device)
        eng.forward(x, sig, cond, eng.cond_stride, 0.0, K._native.PREC_FP32)
        h, w = U.level_hw(mcfg, H, W, level)
        assert eng.tap_count() == B * h * w * c, (tap, eng.tap_count(), (B, h, w, c))
        got = buf[: B * h * w * c].view(B, h, w, c).permute(0, 3, 1, 2).cpu().double()
        assert torch.isfinite(got).all(), tap
        return got

    s0, p = mcfg.get("skip_stages", 0), mcfg["patch_size"]
    got_pin = run_tap("patch_in", s0, mcfg["channels"][max(0, s0 - 1)])
    x64 = x.cpu().double()
    want_pin = F.conv2d(F.pixel_unshuffle(x64, p) if p > 1 else x64, sd64["proj_in.weight"], sd64["proj_in.bias"])
    assert_close(got_pin, want_pin, rtol=1e-4, atol=1e-5, what=f"{name} patch_in")
    outs = {"patch_in": got_pin}
    for tap, (src, op, skip, level) in U.stage_plan(mcfg).items():
        inp = outs[src] if skip is None else torch.cat([outs[src], outs[skip]], dim=1)
        want = U.stage_op(sd64, op, inp, c64)
        got = run_tap(tap, level, want.shape[1])
        assert_close(got, want, rtol=1e-3, atol=1e-4, what=f"{name} stage {tap}")
        outs[tap] = got
    return len(outs)


@pytest.mark.parametrize("name", ["mnist", "cifar10"])
def test_every_stage_against_the_oracle(name):
    """conv3x3 at borders on 28/14/7 and 32/16/8 grids, the skip conv with c_in != c_out on the two-source concat, AdaGN, attention,
    down- and upsampling, patch-in"""
    cfg, sd, model, _ = build(name)
    mcfg = cfg["model"]
    B, (H, W) = 2, mcfg["input_size"]
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, mcfg["input_channels"], H, W, generator=g).to(DEV)
    sig = torch.tensor([0.7, 9.0], device=DEV)
    aug = (torch.randn(B, 9, generator=g) * 0.5).to(DEV)
    check_every_stage(name, cfg, sd, model, x, sig, aug)


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
