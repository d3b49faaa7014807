"""The learned-variance path of image_v1 U-Net models on the H100: kdb_unet_forward_variance's logvar and kdb_variance_loss against float64,
return_variance at fp32, tf32 and fp16, and DenoiserWithVariance.loss's parameter gradients (kdb_unet_forward_train_variance) against the
oracle's float64 autograd, within 8x the oracle's own fp32-vs-float64 distance, bare, in the augment wrapper and in DistributedDataParallel."""
import datetime
import json
import socket
from pathlib import Path

import pytest
import torch

from conftest import load_npz, synth_sd
from oracle import unet_variance_oracle as V
from test_gpu_unet_train import BUFFERS, inputs

import k_diffusion as K

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden"
META = json.loads((GOLDEN / "unet_variance_meta.json").read_text())
VARIANCE = json.loads((GOLDEN / "unet_edges.json").read_text())["variance"]["config"]       # augment wrapper, patch 1
PATCH2 = META["configs"]["patch2_mcond"]                                                      # bare, patch 2, mapping_cond


def build(cfg, seed=3):
    """(cfg, innermost model, its state dict, DenoiserWithVariance around the model make_model returns)"""
    cfg = K.config.load_config(json.loads(json.dumps(cfg)))
    cfg["model"]["dropout_rate"] = 0.0
    model = K.config.make_model(cfg)
    inner = model.inner_model if isinstance(model, K.augmentation.KarrasAugmentWrapper) else model
    sd = synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, seed)
    inner.load_state_dict(sd)
    model = model.cuda().eval()
    den = K.config.make_denoiser_wrapper(cfg)(model)
    assert type(den) is K.layers.DenoiserWithVariance
    return cfg, inner, sd, den


def native_grads(den, inner, x, noise, sigma, kw, gw):
    inner.zero_grad(set_to_none=True)
    loss = den.loss(x.cuda(), noise.cuda(), sigma.cuda(), **{k: v.cuda() for k, v in kw.items()})
    assert loss.grad_fn is not None
    (loss * gw.cuda()).sum().backward()
    return loss.detach().cpu(), {k: p.grad.detach().cpu().clone() for k, p in inner.named_parameters() if p.grad is not None}


def oracle_forward(cfg, params, x, sigma, kw):
    m = cfg["model"]
    fn = V.augment_forward if m.get("augment_wrapper", True) else V.model_forward
    return fn(params, m, x, sigma, **kw)


def oracle_grads(cfg, sd, x, noise, sigma, kw, gw, dtype):
    """layers.py:93-101 around the oracle's U-Net under autograd (losses, logvar and gradients on the CPU)"""
    m = cfg["model"]
    params = {k: v.to(dtype).requires_grad_(not k.endswith(BUFFERS)) for k, v in sd.items()}
    x, noise, sigma, gw = (t.to(dtype) for t in (x, noise, sigma, gw))
    kw = {k: v.to(dtype) for k, v in kw.items()}
    c_in = (1 / (sigma ** 2 + m["sigma_data"] ** 2) ** 0.5).view(-1, 1, 1, 1)
    f, lv = oracle_forward(cfg, params, (x + noise * sigma.view(-1, 1, 1, 1)) * c_in, sigma, kw)
    loss = V.variance_loss(f, lv, x, noise, sigma, m["sigma_data"])
    (loss * gw).sum().backward()
    return loss.detach(), lv.detach(), {k: p.grad for k, p in params.items() if p.requires_grad and p.grad is not None}


def check_against_oracle(cfg, sd, got_loss, got, x, noise, sigma, kw, gw, budget=None):
    """as test_gpu_unet_train.check_against_oracle, for DenoiserWithVariance's loss"""
    l64, _, g64 = oracle_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float64)
    l32, _, g32 = oracle_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float32)
    assert (got_loss.double() - l64).norm() <= 8 * (l32.double() - l64).norm() + 1e-6 * l64.norm()
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
        if budget is not None:
            ref = max(ref, budget[k]["fp32_rel"])
        assert err <= 8 * ref + 1e-6, f"{k}: rel-L2 {err:.3e} vs the fp32 distance {ref:.3e}"


# ------------------------------------------------------------------------------------------------------------------------------
# the two kernels
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,n,lv_scale", [(1, 3 * 8 * 8, 1.0), (5, 3 * 32 * 32, 20.0), (3, 1000, 8.0)])
def test_variance_loss_kernel_against_float64(B, n, lv_scale):
    g = torch.Generator().manual_seed(B * 31 + n)
    x, noise, f = (torch.randn(B, n, generator=g) for _ in range(3))
    sigma = torch.exp(torch.randn(B, generator=g) * 1.5)
    logvar = (torch.rand(B, generator=g) * 2 - 1) * lv_scale
    if B > 1:
        logvar[0], logvar[-1] = lv_scale, -lv_scale
    sd = 0.5
    loss, cot, dlv = K._native.variance_loss(*(t.cuda() for t in (x, noise, sigma)), sd, f.cuda(), logvar.cuda())
    c_skip, c_out = (sd ** 2 / (sigma.double() ** 2 + sd ** 2)).view(-1, 1), (sigma.double() * sd / (sigma.double() ** 2 + sd ** 2) ** 0.5).view(-1, 1)
    x64, n64, f64, lv64 = x.double(), noise.double(), f.double(), logvar.double()
    r = f64 - (x64 - c_skip * (x64 + n64 * sigma.double().view(-1, 1))) / c_out
    m = (r ** 2).mean(1)
    q = m * torch.exp(-lv64)
    want_loss, want_dlv = (q + lv64) / 2, (1 - q) / 2
    want_cot = r * torch.exp(-lv64).view(-1, 1) / n
    assert ((loss.cpu().double() - want_loss).abs() <= 1e-5 * (q.abs() + lv64.abs()) / 2 + 1e-30).all()
    assert ((dlv.cpu().double() - want_dlv).abs() <= 1e-5 * (1 + q) / 2).all()
    assert ((cot.cpu().double() - want_cot).abs() <= 1e-5 * want_cot.abs() + 1e-6 * want_cot.abs().amax(1, keepdim=True)).all()
    again = K._native.variance_loss(*(t.cuda() for t in (x, noise, sigma)), sd, f.cuda(), logvar.cuda())
    assert all(torch.equal(a, b) for a, b in zip((loss, cot, dlv), again))


@pytest.mark.parametrize("cfg", [VARIANCE, PATCH2], ids=["variance", "patch2_mcond"])
def test_logvar_against_float64(cfg):
    """logvar of kdb_unet_forward_variance at fp32 within 8x the oracle's fp32 distance from float64; its output bit for bit the forward's"""
    cfg, inner, sd, den = build(cfg)
    x, _, sigma, kw, _ = inputs(cfg, 4, 31)
    out, lv = den.inner_model(x.cuda(), sigma.cuda(), **{k: v.cuda() for k, v in kw.items()}, return_variance=True)
    assert torch.equal(out, den.inner_model(x.cuda(), sigma.cuda(), **{k: v.cuda() for k, v in kw.items()}))
    p64 = {k: v.double() for k, v in sd.items()}
    p32 = {k: v.float() for k, v in sd.items()}
    _, lv64 = oracle_forward(cfg, p64, x.double(), sigma.double(), {k: v.double() for k, v in kw.items()})
    _, lv32 = oracle_forward(cfg, p32, x, sigma, kw)
    assert lv.shape == (4,) and lv.dtype == torch.float32
    err, ref = (lv.cpu().double() - lv64).abs(), (lv32.double() - lv64).abs()
    assert (err <= 8 * ref.max() + 1e-6 * lv64.abs().max()).all(), (err, ref)


@pytest.mark.parametrize("precision", ["fp32", "tf32", "fp16"])
def test_return_variance_at_every_precision(precision):
    """return_variance's first element is bit for bit the plain forward at that precision, bare and through the augment wrapper; logvar
    comes from the same features and stays near the float64 oracle's"""
    for cfg in (VARIANCE, PATCH2):
        cfg, inner, sd, den = build(cfg)
        model = den.inner_model.set_precision(precision)
        x, _, sigma, kw, _ = inputs(cfg, 3, 32)
        x, sigma, kw = x.cuda(), sigma.cuda(), {k: v.cuda() for k, v in kw.items()}
        out, lv = model(x, sigma, **kw, return_variance=True)
        assert torch.equal(out, model(x, sigma, **kw))
        _, lv64 = oracle_forward(cfg, {k: v.double() for k, v in sd.items()}, x.cpu().double(), sigma.cpu().double(),
                                 {k: v.cpu().double() for k, v in kw.items()})
        tol = 1e-5 if precision == "fp32" else 2e-2
        assert ((lv.cpu().double() - lv64).abs() <= tol * (1 + lv64.abs())).all(), (precision, lv, lv64)
        again = model(x, sigma, **kw, return_variance=True)
        assert torch.equal(again[0], out) and torch.equal(again[1], lv)


# ------------------------------------------------------------------------------------------------------------------------------
# DenoiserWithVariance.loss's gradients
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("cfg", [VARIANCE, PATCH2], ids=["wrapped", "bare"])
def test_gradients_match_float64(cfg, B):
    cfg, inner, sd, den = build(cfg)
    x, noise, sigma, kw, gw = inputs(cfg, B, 40 + B)
    loss, got = native_grads(den, inner, x, noise, sigma, kw, gw)
    assert set(got) == {k for k, _ in inner.named_parameters()}
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw)


@pytest.mark.parametrize("name", sorted(META["cases"]))
def test_recorded_reference_cases(name):
    """The reference's DenoiserWithVariance.loss (oracle/make_golden_unet_variance.py): logvar and the losses against its float64 ones,
    every gradient within 8x the larger of the oracle's and the reference's own fp32 distance"""
    rec = load_npz("unet_variance.npz")
    cfg, inner, sd, den = build(META["configs"][name])
    x, noise, sigma = rec[f"{name}_x"], rec[f"{name}_noise"], rec[f"{name}_sigma"]
    kw = {k: rec[f"{name}_{k}"] for k in ("aug_cond", "mapping_cond") if f"{name}_{k}" in rec}
    gw = torch.ones(x.shape[0])
    loss, got = native_grads(den, inner, x, noise, sigma, kw, gw)
    l64, l32 = rec[f"{name}_loss_float64"], rec[f"{name}_loss_float32"]
    assert (loss.double() - l64).norm() <= 8 * (l32 - l64).norm() + 1e-6 * l64.norm()
    c_in = (1 / (sigma ** 2 + cfg["model"]["sigma_data"] ** 2) ** 0.5).view(-1, 1, 1, 1)
    _, lv = den.inner_model(((x + noise * sigma.view(-1, 1, 1, 1)) * c_in).cuda(), sigma.cuda(), **{k: v.cuda() for k, v in kw.items()},
                            return_variance=True)
    lv64, lv32 = rec[f"{name}_logvar_float64"], rec[f"{name}_logvar_float32"]
    assert (lv.cpu().double() - lv64).abs().max() <= 8 * (lv32 - lv64).abs().max() + 1e-6 * lv64.abs().max()
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw, budget=META["cases"][name])


def test_variance_row_gets_its_gradient_and_plain_denoiser_leaves_it_zero():
    cfg, inner, sd, den = build(VARIANCE)
    x, noise, sigma, kw, gw = inputs(cfg, 3, 50)
    _, got = native_grads(den, inner, x, noise, sigma, kw, gw)
    _, _, g64 = oracle_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float64)
    for k in ("proj_out.weight", "proj_out.bias"):
        row, want = got[k][-1].double(), g64[k][-1]
        assert (row != 0).all() and (row - want).norm() <= 1e-4 * want.norm(), k
    plain = K.layers.Denoiser(den.inner_model, cfg["model"]["sigma_data"])
    _, pg = native_grads(plain, inner, x, noise, sigma, kw, gw)
    assert (pg["proj_out.weight"][-1] == 0).all() and pg["proj_out.bias"][-1] == 0


def test_two_calls_bit_identical_and_batch_is_sum_of_images():
    cfg, inner, sd, den = build(PATCH2)
    x, noise, sigma, kw, gw = inputs(cfg, 4, 51)
    l1, g1 = native_grads(den, inner, x, noise, sigma, kw, gw)
    l2, g2 = native_grads(den, inner, x, noise, sigma, kw, gw)
    assert torch.equal(l1, l2) and all(torch.equal(g1[k], g2[k]) for k in g1)
    parts = [native_grads(den, inner, x[i:i + 1], noise[i:i + 1], sigma[i:i + 1], {k: v[i:i + 1] for k, v in kw.items()}, gw[i:i + 1])
             for i in range(4)]
    assert torch.allclose(torch.cat([p[0] for p in parts]), l1, rtol=1e-6, atol=0)
    for k in g1:
        total = sum(p[1][k].double() for p in parts)
        assert (g1[k].double() - total).norm().item() <= 1e-5 * total.norm().item() + 1e-7, k


def test_frozen_parameters_leave_the_others_bit_identical():
    cfg, inner, sd, den = build(VARIANCE)
    x, noise, sigma, kw, gw = inputs(cfg, 2, 52)
    _, full = native_grads(den, inner, x, noise, sigma, kw, gw)
    frozen = [k for k in full if "d_blocks" in k or k.startswith("mapping") or k == "proj_out.bias"]
    for k, p in inner.named_parameters():
        p.requires_grad_(k not in frozen)
    _, part = native_grads(den, inner, x, noise, sigma, kw, gw)
    assert set(part) == set(full) - set(frozen)
    assert all(torch.equal(part[k], full[k]) for k in part)


def test_adamw_step_on_param_groups_matches_oracle():
    """as test_gpu_unet_train's: the native AdamW step equals the oracle's to a small fraction of lr wherever |g| is firm"""
    cfg, inner, sd, den = build(PATCH2)
    x, noise, sigma, kw, gw = inputs(cfg, 2, 53)
    lr = 1e-3
    names = {id(p): k for k, p in inner.named_parameters()}
    opt = torch.optim.AdamW(den.inner_model.param_groups(lr), betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-2)
    native_grads(den, inner, x, noise, sigma, kw, gw)
    opt.step()
    ref = {k: v.double().clone().requires_grad_(not k.endswith(BUFFERS)) for k, v in sd.items()}
    _, _, g64 = oracle_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float64)
    for k, g in g64.items():
        ref[k].grad = g
    torch.optim.AdamW([dict(g, params=[ref[names[id(p)]] for p in g["params"]]) for g in inner.param_groups(lr)], betas=(0.9, 0.95), eps=1e-6,
                      weight_decay=1e-2).step()
    for k, p in inner.named_parameters():
        want = ref[k].detach()
        err = (p.detach().cpu().double() - want).abs()
        firm = g64[k].abs() > 1e-4 * g64[k].abs().max() + 1e-5
        assert (err[firm] <= 1e-3 * lr + 2e-7 * want.abs()[firm]).all(), k
        assert (err <= 2 * lr + 2e-7 * want.abs()).all(), k


def test_train_loop_loss_falls():
    """train.py's loop on a has_variance config: make_denoiser_wrapper, loss, backward, AdamW on param_groups, ema_update -- 20 native
    steps on one fixed batch, the mean loss falling"""
    cfg, inner, sd, den = build(VARIANCE)
    ema = K.config.make_model(cfg).cuda().eval()
    ema.inner_model.load_state_dict(sd)
    x, noise, sigma, kw, _ = inputs(cfg, 8, 54)
    x, noise, sigma, kw = x.cuda(), noise.cuda(), sigma.cuda(), {k: v.cuda() for k, v in kw.items()}
    opt = torch.optim.AdamW(den.inner_model.param_groups(1e-3), betas=(0.95, 0.999), eps=1e-6, weight_decay=1e-3)
    launches = K._native.launch_count()
    losses = []
    for _ in range(20):
        opt.zero_grad(set_to_none=True)
        loss = den.loss(x, noise, sigma, **kw).mean()
        loss.backward()
        opt.step()
        K.utils.ema_update(den.inner_model, ema, 0.99)
        losses.append(loss.item())
    assert K._native.launch_count() > launches
    assert all(map(lambda v: v == v, losses)) and losses[-1] < 0.9 * losses[0], losses


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_ddp_world_size_one_is_the_unwrapped_step():
    """DenoiserWithVariance.loss around DistributedDataParallel (gloo, one rank): the native loss runs inside DDP's forward, and the loss
    and every gradient equal the unwrapped model's, bit for bit"""
    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel as DDP
    cfg, inner, sd, den = build(VARIANCE)
    x, noise, sigma, kw, gw = inputs(cfg, 4, 55)
    l_solo, g_solo = native_grads(den, inner, x, noise, sigma, kw, gw)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1,
                            timeout=datetime.timedelta(minutes=5))
    try:
        cfg, inner, sd, den = build(VARIANCE)
        ddp = DDP(den.inner_model, device_ids=[torch.cuda.current_device()])
        dden = K.config.make_denoiser_wrapper(cfg)(ddp)
        assert dden.is_native() and isinstance(dden.inner_model, DDP)
        l_ddp, g_ddp = native_grads(dden, inner, x, noise, sigma, kw, gw)
    finally:
        dist.destroy_process_group()
    assert torch.equal(l_solo, l_ddp)
    assert set(g_solo) == set(g_ddp) and all(torch.equal(g_solo[k], g_ddp[k]) for k in g_solo)
