"""Parameter gradients of image_v1 U-Net models on the H100 (Denoiser.loss, kdb_unet_forward_train): every parameter's native gradient
against the oracle's float64 autograd, within 8x the oracle's own fp32-vs-float64 distance; exact zeros where the float64 gradient is
exactly zero; bits stable across calls; a batch equal to the sum of its images; frozen parameters; the loss forward against the sampling
forward; one AdamW step on param_groups."""
import json
from pathlib import Path

import pytest
import torch

from conftest import synth_sd
from oracle import unet_oracle as U
from oracle import kdiff_oracle as O

import k_diffusion as K

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden"
EDGES = json.loads((GOLDEN / "unet_edges.json").read_text())
CONFIGS = json.loads((GOLDEN / "unet_configs.json").read_text())
BUFFERS = ("timestep_embed.weight", ".kernel")

# two levels, self-attention on the inner one, a 1x1 skip conv and an identity skip, no augment wrapper
SMALL = {"model": {"type": "image_v1", "input_channels": 3, "input_size": [16, 16], "mapping_out": 32, "depths": [1, 2], "channels": [32, 64],
                   "self_attn_depths": [False, True], "augment_wrapper": False, "sigma_data": 0.5, "dropout_rate": 0.0}}


def build(cfg, seed=3, weights=True):
    cfg = K.config.load_config(cfg)
    model = K.config.make_model(cfg)
    inner = model.inner_model if isinstance(model, K.augmentation.KarrasAugmentWrapper) else model
    sd = {k: v.clone() for k, v in inner.state_dict().items()}
    if weights:
        sd = synth_sd({k: list(v.shape) for k, v in sd.items()}, seed)
        inner.load_state_dict(sd)
    model = model.cuda().eval()
    m = cfg["model"]
    if m["has_variance"]:   # the reference's Denoiser around a has_variance model: its loss drops the variance channel
        return cfg, inner, sd, K.layers.Denoiser(model, m["sigma_data"], weighting=m["loss_weighting"])
    return cfg, inner, sd, K.config.make_denoiser_wrapper(cfg)(model)


def inputs(cfg, B, seed):
    m = cfg["model"]
    H, W = m["input_size"]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, m["input_channels"], H, W, generator=g) * 0.5
    noise = torch.randn(x.shape, generator=g)
    sigma = torch.exp(torch.randn(B, generator=g) * 1.2 - 0.4)
    kw = {}
    wrap = m.get("augment_wrapper", True)
    if wrap:
        kw["aug_cond"] = torch.randn(B, 9, generator=g) * 0.3
    user = m["mapping_cond_dim"]
    if user:
        kw["mapping_cond"] = torch.randn(B, user, generator=g)
    gw = torch.rand(B, generator=g) + 0.5
    return x, noise, sigma, kw, gw


def native_grads(model, inner, x, noise, sigma, kw, gw):
    inner.zero_grad(set_to_none=True)
    loss = model.loss(x.cuda(), noise.cuda(), sigma.cuda(), **{k: v.cuda() for k, v in kw.items()})
    assert loss.grad_fn is not None
    (loss * gw.cuda()).sum().backward()
    return loss.detach().cpu(), {k: p.grad.detach().cpu().clone() for k, p in inner.named_parameters() if p.grad is not None}


def oracle_grads(cfg, sd, x, noise, sigma, kw, gw, dtype, simple=False, device="cpu"):
    """layers.py:76-86 (or :107-111) around the oracle's U-Net, autograd on `device` (losses and gradients returned on the CPU)"""
    m = cfg["model"]
    params = {k: v.to(device, dtype).requires_grad_(not k.endswith(BUFFERS)) for k, v in sd.items()}
    x, noise, sigma, gw = (t.to(device, dtype) for t in (x, noise, sigma, gw))
    kw = {k: v.to(device, dtype) for k, v in kw.items()}
    sd_ = m["sigma_data"]
    c_skip, c_out, c_in = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sigma, sd_)]
    s4 = sigma.view(-1, 1, 1, 1)
    noised = x + noise * s4
    fn = U.augment_forward if m.get("augment_wrapper", True) else U.model_forward
    f = fn(params, m, noised * c_in, sigma, **kw)
    if simple:
        den = f * c_out + noised * c_skip
        loss = (((noised - den) / s4 - noise) ** 2).flatten(1).mean(1)
    else:
        w = (sigma * sd_) ** 2 / (sigma ** 2 + sd_ ** 2) ** 2 if m["loss_weighting"] == "soft-min-snr" else torch.ones_like(sigma)
        loss = ((f - (x - c_skip * noised) / c_out) ** 2).flatten(1).mean(1) * w
    (loss * gw).sum().backward()
    return loss.detach().cpu(), {k: p.grad.cpu() for k, p in params.items() if p.requires_grad and p.grad is not None}


def check_against_oracle(cfg, sd, got_loss, got, x, noise, sigma, kw, gw, simple=False, budget=None, device="cpu"):
    """Each native gradient within 8x the fp32-vs-float64 distance of the oracle's gradient, plus 1e-6 relative; exactly 0 where the
    float64 gradient is exactly 0.  The key rows of qkv_proj's bias are left out of the zero check: softmax does not change when one key
    bias is added to every score of a query, so their gradient is 0 only through cancellation, which fp32 leaves at rounding level."""
    l64, g64 = oracle_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float64, simple, device)
    l32, g32 = oracle_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float32, simple, device)
    assert torch.allclose(got_loss.double(), l64, rtol=1e-4, atol=0)
    assert set(got) == set(g64), set(got) ^ set(g64)
    for k, want in g64.items():
        zero = want == 0
        if k.endswith("qkv_proj.bias"):
            zero[want.numel() // 3:2 * want.numel() // 3] = False
        assert (got[k][zero] == 0).all(), f"{k}: nonzero where the float64 gradient is exactly zero"
        scale = want.norm().item()
        if scale == 0:
            continue
        err = (got[k].double() - want).norm().item() / scale
        ref = (g32[k].double() - want).norm().item() / scale
        if budget is not None:   # the reference's own recorded fp32 distance, where the inputs are the recording's
            ref = max(ref, budget[k]["fp32_rel"])
        assert err <= 8 * ref + 1e-6, f"{k}: rel-L2 {err:.3e} vs the fp32 distance {ref:.3e}"


@pytest.mark.parametrize("weighting,simple", [("karras", False), ("soft-min-snr", False), ("karras", True)])
def test_small_unet_gradients_match_float64(weighting, simple):
    cfg, inner, sd, model = build({"model": dict(SMALL["model"], loss_weighting=weighting, loss_config="simple" if simple else "karras")})
    assert isinstance(model, K.layers.SimpleLossDenoiser) == simple
    x, noise, sigma, kw, gw = inputs(cfg, 3, 0)
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw, simple)


@pytest.mark.parametrize("name", sorted(EDGES))
def test_edge_config_gradients_match_float64(name):
    cfg, inner, sd, model = build(EDGES[name]["config"])
    x, noise, sigma, kw, gw = inputs(cfg, 2, 1)
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw)
    if cfg["model"]["has_variance"]:
        assert (got["proj_out.weight"][-1] == 0).all() and got["proj_out.bias"][-1] == 0


@pytest.mark.parametrize("name", ["mnist", "cifar10"])
def test_reference_configs_gradients_match_float64(name):
    cfg, inner, sd, model = build(CONFIGS[name]["config"])
    x, noise, sigma, kw, gw = inputs(cfg, 2, 2)
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    assert set(got) == {k for k, p in inner.named_parameters()}
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw)


@pytest.fixture(scope="module")
def no_tf32():
    """cuDNN convolutions and cuBLAS matmuls at full fp32 for the oracle on the GPU: under TF32 (operands rounded to 2^-11 instead of 2^-24)
    its fp32-vs-float64 distance, and with it the gate, would loosen by three to four orders of magnitude"""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.mark.parametrize("name", ["mnist", "cifar10"])
def test_reference_configs_at_the_training_batch_size(name, no_tf32):
    """train.py's default batch of 64, where every level's weight gradients run several row chunks: every gradient within 8x the oracle's
    fp32 distance (the oracle run on the GPU in float64 and fp32); every element of every gradient written through forward_train into NaN;
    the batch equal to the float64 sum of eight batches of 8; two calls bit-identical"""
    assert not torch.backends.cudnn.allow_tf32 and not torch.backends.cuda.matmul.allow_tf32
    cfg, inner, sd, model = build(CONFIGS[name]["config"])
    B = 64
    x, noise, sigma, kw, gw = inputs(cfg, B, 15)
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    assert set(got) == {k for k, p in inner.named_parameters()}
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw, device="cuda")

    l2, again = native_grads(model, inner, x, noise, sigma, kw, gw)
    assert torch.equal(loss, l2) and all(torch.equal(got[k], again[k]) for k in got), "two calls differ"

    parts = [native_grads(model, inner, x[i:i + 8], noise[i:i + 8], sigma[i:i + 8], {k: v[i:i + 8] for k, v in kw.items()}, gw[i:i + 8])[1]
             for i in range(0, B, 8)]
    for k in got:
        total = sum(p[k].double() for p in parts)
        assert (got[k].double() - total).norm().item() <= 1e-5 * total.norm().item() + 1e-7, k

    augment = cfg["model"].get("augment_wrapper", True)
    kwc = {k: v.cuda() for k, v in kw.items()}
    ev = inner.native_eval(x.cuda(), sigma.cuda(), kwc.get("aug_cond"), mapping_cond=kwc.get("mapping_cond"), precision=K._native.PREC_FP32,
                           augment=augment)
    grads = {k: torch.full_like(p, float("nan")) for k, p in inner.named_parameters()}
    ev.engine.forward_train(ev.x, torch.randn_like(ev.x), ev.sigma, *ev.cond, ev.conditioning(), grads)
    torch.cuda.synchronize()
    for k, g in grads.items():
        assert torch.isfinite(g).all(), f"{k}: {int((~torch.isfinite(g)).sum())} elements not written"


def test_reference_init_leaves_only_proj_out_nonzero():
    """At the reference's init every last conv, out_proj and proj_out are zero, so F does not depend on any other parameter's value
    through a nonzero path: every gradient but proj_out's is exactly zero"""
    torch.manual_seed(0)
    cfg, inner, sd, model = build(SMALL, weights=False)
    x, noise, sigma, kw, gw = inputs(cfg, 2, 3)
    _, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    for k, g in got.items():
        if k.startswith("proj_out."):
            assert g.abs().sum() > 0, k
        else:
            assert (g == 0).all(), k


def test_aug_cond_from_the_augmentation_pipeline():
    cfg, inner, sd, model = build(EDGES["mcond_aug"]["config"])
    m = cfg["model"]
    B = 2
    imgs = torch.randint(0, 256, (B, m["input_channels"], m["input_size"][0], m["input_size"][1]), dtype=torch.uint8,
                         generator=torch.Generator().manual_seed(5)).cuda()
    image, _, aug_cond = K.augmentation.KarrasAugmentationPipeline(1.0).augment(imgs)
    x, noise, sigma, kw, gw = inputs(cfg, B, 4)
    x, kw["aug_cond"] = image.float().cpu(), aug_cond.float().cpu()
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw)


def test_two_calls_bit_identical_and_batch_is_sum_of_images():
    cfg, inner, sd, model = build(EDGES["mcond_aug"]["config"])
    x, noise, sigma, kw, gw = inputs(cfg, 3, 6)
    l1, g1 = native_grads(model, inner, x, noise, sigma, kw, gw)
    l2, g2 = native_grads(model, inner, x, noise, sigma, kw, gw)
    assert torch.equal(l1, l2)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k
    parts = [native_grads(model, inner, x[i:i + 1], noise[i:i + 1], sigma[i:i + 1], {k: v[i:i + 1] for k, v in kw.items()}, gw[i:i + 1])[1]
             for i in range(3)]
    for k in g1:
        total = sum(p[k].double() for p in parts)
        scale = total.norm().item()
        assert (g1[k].double() - total).norm().item() <= 1e-5 * scale + 1e-7, k


def test_frozen_parameters_leave_the_others_bit_identical():
    cfg, inner, sd, model = build(SMALL)
    x, noise, sigma, kw, gw = inputs(cfg, 2, 7)
    _, full = native_grads(model, inner, x, noise, sigma, kw, gw)
    frozen = [k for k in full if "d_blocks" in k or k.startswith("mapping")]
    for k, p in inner.named_parameters():
        p.requires_grad_(k not in frozen)
    _, part = native_grads(model, inner, x, noise, sigma, kw, gw)
    assert set(part) == set(full) - set(frozen)
    for k in part:
        assert torch.equal(part[k], full[k]), k


def test_loss_forward_is_the_sampling_forward():
    """The loss's F is kdb_unet_forward at fp32, and forward_train's out is that bit for bit"""
    cfg, inner, sd, model = build(EDGES["identity_concat"]["config"])
    x, noise, sigma, kw, gw = inputs(cfg, 2, 8)
    x, sig = x.cuda(), sigma.cuda()
    kw = {k: v.cuda() for k, v in kw.items()}
    augment = cfg["model"].get("augment_wrapper", True)
    ev = inner.native_eval(x, sig, kw.get("aug_cond"), mapping_cond=kw.get("mapping_cond"), precision=K._native.PREC_FP32, augment=augment)
    eng = ev.engine
    cond = ev.conditioning()
    f = eng.train_forward(ev.x, ev.sigma, cond, eng.cond_stride, 0.0, K._native.PREC_FP32)
    assert torch.equal(f, inner.native_eval(x, sig, kw.get("aug_cond"), mapping_cond=kw.get("mapping_cond"), augment=augment).forward(0.0))
    grads = {k: torch.empty_like(p) for k, p in inner.named_parameters()}
    out = eng.forward_train(ev.x, torch.randn_like(ev.x), ev.sigma, *ev.cond, cond, grads)
    assert torch.equal(out, f)


def test_adamw_step_on_param_groups_matches_oracle():
    """Adam's first step moves each element by lr g / (|g| + eps) plus the decay: wherever |g| is well above eps and the gradients' fp32
    error, the native step must equal the oracle's to a small fraction of lr; elsewhere by at most the 2 lr a flipped sign could cost"""
    cfg, inner, sd, model = build(SMALL)
    x, noise, sigma, kw, gw = inputs(cfg, 2, 9)
    lr = 1e-3
    names = {id(p): k for k, p in inner.named_parameters()}
    opt = torch.optim.AdamW(inner.param_groups(lr), betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-2)
    native_grads(model, inner, x, noise, sigma, kw, gw)
    opt.step()
    ref = {k: v.double().clone().requires_grad_(not k.endswith(BUFFERS)) for k, v in sd.items()}
    groups = [dict(g, params=[ref[names[id(p)]] for p in g["params"]]) for g in inner.param_groups(lr)]
    _, g64 = oracle_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float64)
    for k, g in g64.items():
        ref[k].grad = g
    torch.optim.AdamW(groups, betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-2).step()
    for k, p in inner.named_parameters():
        want = ref[k].detach()
        err = (p.detach().cpu().double() - want).abs()
        firm = g64[k].abs() > 1e-4 * g64[k].abs().max() + 1e-5
        assert firm.any(), k
        assert (err[firm] <= 1e-3 * lr + 2e-7 * want.abs()[firm]).all(), k
        assert (err <= 2 * lr + 2e-7 * want.abs()).all(), k


META = json.loads((GOLDEN / "unet_train_meta.json").read_text())


@pytest.mark.parametrize("name", sorted(META["cases"]))
def test_recorded_reference_cases(name):
    """The reference's recorded cases (oracle/make_golden_unet_train.py): the native loss against the reference's float64 loss, every
    gradient within 8x the larger of the oracle's and the reference's own fp32 distance"""
    from conftest import load_npz
    rec = load_npz("unet_train.npz")
    cfg, inner, sd, model = build(META["configs"][name])
    x, noise, sigma = rec[f"{name}_x"], rec[f"{name}_noise"], rec[f"{name}_sigma"]
    kw = {k: rec[f"{name}_{k}"] for k in ("aug_cond", "mapping_cond") if f"{name}_{k}" in rec}
    gw = torch.ones(x.shape[0])
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    assert torch.allclose(loss.double(), rec[f"{name}_loss_float64"].double(), rtol=1e-4, atol=0)
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw, budget=META["cases"][name])


def test_gradients_after_an_optimizer_step_are_those_of_the_updated_weights():
    """After AdamW updates the weights in place, the next loss rebinds the engine and rebuilds the flipped input-gradient weights: its
    gradients equal, bit for bit, those of a fresh model loaded with the updated weights"""
    cfg, inner, sd, model = build(EDGES["mcond_aug"]["config"])
    x, noise, sigma, kw, gw = inputs(cfg, 2, 10)
    opt = torch.optim.AdamW(inner.param_groups(1e-2), betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-2)
    native_grads(model, inner, x, noise, sigma, kw, gw)
    opt.step()
    l1, g1 = native_grads(model, inner, x, noise, sigma, kw, gw)
    _, fresh, _, fmodel = build(EDGES["mcond_aug"]["config"])
    fresh.load_state_dict(inner.state_dict())
    l2, g2 = native_grads(fmodel, fresh, x, noise, sigma, kw, gw)
    assert torch.equal(l1, l2)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k


def test_train_loop_matches_the_oracle():
    """Ten train.py-shaped steps (augment, loss, backward, AdamW on param_groups, ema_update) next to the same loop on the oracle under
    torch autograd in float64 and fp32: per-step losses and the final EMA weights within 8x the oracle's own fp32-vs-float64 distance"""
    cfg, inner, sd, model = build(EDGES["mcond_aug"]["config"])
    m = cfg["model"]
    ema = K.config.make_model(cfg).cuda().eval()
    ema.inner_model.load_state_dict(sd)
    B, steps, lr, decay = 4, 10, 2e-4, 0.9
    g = torch.Generator().manual_seed(12)
    imgs = torch.randint(0, 256, (B, m["input_channels"], *m["input_size"]), dtype=torch.uint8, generator=g).cuda()
    pipe = K.augmentation.KarrasAugmentationPipeline(0.5)
    batches = []
    for i in range(steps):
        image, _, aug = pipe.augment(imgs, generator=torch.Generator(device="cuda").manual_seed(i))
        batches.append((image.cpu(), aug.cpu(), torch.randn(image.shape, generator=g), torch.exp(torch.randn(B, generator=g) * 1.2 - 0.4),
                        torch.randn(B, m["mapping_cond_dim"], generator=g)))
    opt = torch.optim.AdamW(inner.param_groups(lr), betas=(0.95, 0.999), eps=1e-6, weight_decay=1e-3)
    native_losses = []
    for x, aug, noise, sigma, mc in batches:
        opt.zero_grad(set_to_none=True)
        loss = model.loss(x.cuda(), noise.cuda(), sigma.cuda(), aug_cond=aug.cuda(), mapping_cond=mc.cuda())
        loss.mean().backward()
        opt.step()
        K.utils.ema_update(inner, ema.inner_model, decay)
        native_losses.append(loss.detach().cpu().double())
    names = {id(p): k for k, p in inner.named_parameters()}

    def oracle_loop(dtype):
        params = {k: v.to(dtype).clone().requires_grad_(not k.endswith(BUFFERS)) for k, v in sd.items()}
        avg = {k: v.detach().clone() for k, v in params.items()}
        topt = torch.optim.AdamW([dict(gr, params=[params[names[id(p)]] for p in gr["params"]]) for gr in inner.param_groups(lr)],
                                 betas=(0.95, 0.999), eps=1e-6, weight_decay=1e-3)
        losses = []
        for x, aug, noise, sigma, mc in batches:
            topt.zero_grad(set_to_none=True)
            x, aug, noise, sigma, mc = (t.to(dtype) for t in (x, aug, noise, sigma, mc))
            c_skip, c_out, c_in = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sigma, m["sigma_data"])]
            noised = x + noise * sigma.view(-1, 1, 1, 1)
            f = U.augment_forward(params, m, noised * c_in, sigma, aug_cond=aug, mapping_cond=mc)
            sd_ = m["sigma_data"]
            w = (sigma * sd_) ** 2 / (sigma ** 2 + sd_ ** 2) ** 2
            loss = ((f - (x - c_skip * noised) / c_out) ** 2).flatten(1).mean(1) * w
            loss.mean().backward()
            topt.step()
            with torch.no_grad():
                for k, p in params.items():
                    avg[k].lerp_(p, 1 - decay) if p.requires_grad else avg[k].copy_(p)
            losses.append(loss.detach().double())
        return losses, {k: v.double() for k, v in avg.items()}

    l64, a64 = oracle_loop(torch.float64)
    l32, a32 = oracle_loop(torch.float32)
    for got, want, w32 in zip(native_losses, l64, l32):
        assert (got - want).norm() <= 8 * (w32 - want).norm() + 1e-6 * want.norm()
    got_avg = {k: v.detach().cpu().double() for k, v in ema.inner_model.state_dict().items()}
    for k, want in a64.items():
        scale = want.norm().item()
        err, ref = (got_avg[k] - want).norm().item() / scale, (a32[k] - want).norm().item() / scale
        assert err <= 8 * ref + 1e-6, f"{k}: rel-L2 {err:.3e} vs the fp32 distance {ref:.3e}"


def test_unused_parameters_get_no_gradient_and_are_refused_by_the_abi():
    """Without mapping_cond, a bare model never uses mapping_cond.weight; below skip_stages, the blocks never run: no gradient for either,
    as under torch, and kdb_unet_set_grad refuses the skipped blocks' keys"""
    cfg, inner, sd, model = build(EDGES["mcond_plain"]["config"])
    assert not cfg["model"].get("augment_wrapper", True)
    x, noise, sigma, kw, gw = inputs(cfg, 2, 13)
    kw.pop("mapping_cond")
    _, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    assert "mapping_cond.weight" not in got and inner.mapping_cond.weight.grad is None
    check_against_oracle(cfg, sd, *native_grads(model, inner, x, noise, sigma, kw, gw), x, noise, sigma, kw, gw)
    cfg, inner, sd, model = build(EDGES["patch2_skip1"]["config"])
    x, noise, sigma, kw, gw = inputs(cfg, 2, 14)
    _, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    assert not any(k.startswith("u_net.d_blocks.0.") for k in got)
    eng = inner.engine(cfg["model"].get("augment_wrapper", True))
    t = torch.zeros_like(dict(inner.named_parameters())[next(k for k, _ in inner.named_parameters() if k.startswith("u_net.d_blocks.0."))])
    key = next(k for k, _ in inner.named_parameters() if k.startswith("u_net.d_blocks.0."))
    L = K._native.lib()
    dims = (K._native._i64 * t.ndim)(*t.shape)
    assert L.kdb_unet_set_grad(eng._h, key.encode(), K._native.ptr(t), dims, t.ndim) == -1
    assert b"skip_stages" in L.kdb_last_error()
