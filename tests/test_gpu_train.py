"""Parameter gradients of image_transformer_v2 models on the H100 (Denoiser.loss, kdb_model_forward_train): every parameter's native
gradient against the oracle's float64 autograd, within a multiple of the oracle's own fp32-vs-float64 distance; exact zeros where the
float64 gradient is exactly zero; bits stable across calls; a batch equal to the sum of its images; and one AdamW step on param_groups."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from conftest import synth_sd
from oracle import kdiff_oracle as O

import k_diffusion as K

pytestmark = pytest.mark.gpu

# class-conditional, soft-min-snr (the shape of the MNIST config at a test size)
CLASS = {"model": {"type": "image_transformer_v2", "input_channels": 1, "input_size": [16, 16], "patch_size": [2, 2], "depths": [2, 1],
                   "widths": [32, 64], "d_ffs": [64, 96], "mapping_width": 64, "mapping_depth": 2, "mapping_d_ff": 96,
                   "loss_weighting": "soft-min-snr", "sigma_data": 0.6,
                   "self_attns": [{"type": "shifted-window", "d_head": 16, "window_size": 4}, {"type": "global", "d_head": 16}]},
         "dataset": {"num_classes": 10}}
# three levels (shifted-window, neighborhood, none), mapping_cond, aug_cond through the augment wrapper
LEVELS3 = {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [32, 32], "patch_size": [2, 2], "depths": [1, 1, 1],
                     "widths": [32, 48, 64], "d_ffs": [64, 96, 128], "mapping_width": 64, "mapping_depth": 1, "mapping_d_ff": 128,
                     "mapping_cond_dim": 12, "sigma_data": 0.5,
                     "self_attns": [{"type": "shifted-window", "d_head": 16, "window_size": 4},
                                    {"type": "neighborhood", "d_head": 16, "kernel_size": 3}, {"type": "none"}]}}


def build(cfg, wrap=False):
    cfg = K.config.load_config(cfg)
    inner = K.config.make_model(cfg)
    sd = synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, 3)
    inner.load_state_dict(sd)
    inner = inner.cuda().eval()
    model = K.config.make_denoiser_wrapper(cfg)(K.augmentation.KarrasAugmentWrapper(inner) if wrap else inner)
    return cfg, inner, sd, model


def inputs(cfg, B, seed, size=None, classes=None):
    m = cfg["model"]
    H, W = size or m["input_size"]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, m["input_channels"], H, W, generator=g) * 0.5
    noise = torch.randn(x.shape, generator=g)
    sigma = torch.exp(torch.randn(B, generator=g) * 1.2 - 0.4)
    kw = {}
    if cfg["dataset"]["num_classes"]:
        kw["class_cond"] = torch.tensor(classes) if classes is not None else torch.randint(0, cfg["dataset"]["num_classes"], (B,), generator=g)
    if m["mapping_cond_dim"]:
        kw["aug_cond"] = torch.randn(B, 9, generator=g) * 0.3
        kw["mapping_cond"] = torch.randn(B, m["mapping_cond_dim"] - 9, generator=g)
    gw = torch.rand(B, generator=g) + 0.5   # the incoming gradient of each sample's loss
    return x, noise, sigma, kw, gw


def native_grads(model, inner, x, noise, sigma, kw, gw):
    inner.zero_grad(set_to_none=True)
    loss = model.loss(x.cuda(), noise.cuda(), sigma.cuda(), **{k: v.cuda() for k, v in kw.items()})
    assert loss.grad_fn is not None
    (loss * gw.cuda()).sum().backward()
    return loss.detach().cpu(), {k: p.grad.detach().cpu().clone() for k, p in inner.named_parameters()}


def oracle_grads(cfg, sd, x, noise, sigma, kw, gw, dtype, simple=False, device="cpu"):
    """layers.py:76-86 (or :107-111) around the oracle's model, autograd on `device` (losses and gradients returned on the CPU)"""
    m = cfg["model"]
    params = {k: v.to(device, dtype).requires_grad_(not k.endswith(("pos_emb.freqs", "time_emb.weight", "aug_emb.weight")))
              for k, v in sd.items()}
    x, noise, sigma, gw = (t.to(device, dtype) for t in (x, noise, sigma, gw))
    kw = {k: (v.to(device, dtype) if v.is_floating_point() else v.to(device)) for k, v in kw.items()}
    if "aug_cond" in kw:   # the augment wrapper: mapping_cond = cat([aug_cond, mapping_cond])
        kw["mapping_cond"] = torch.cat([kw.pop("aug_cond"), kw["mapping_cond"]], 1)
    sd_ = m["sigma_data"]
    c_skip, c_out, c_in = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sigma, sd_)]
    s4 = sigma.view(-1, 1, 1, 1)
    noised = x + noise * s4
    with torch.device(device):   # the oracle's position tables and masks on the same device
        f = O.model_forward(params, m, noised * c_in, sigma, **kw)
    if simple:
        den = f * c_out + noised * c_skip
        loss = (((noised - den) / s4 - noise) ** 2).flatten(1).mean(1)
    else:
        w = (sigma * sd_) ** 2 / (sigma ** 2 + sd_ ** 2) ** 2 if m["loss_weighting"] == "soft-min-snr" else torch.ones_like(sigma)
        loss = ((f - (x - c_skip * noised) / c_out) ** 2).flatten(1).mean(1) * w
    (loss * gw).sum().backward()
    return loss.detach().cpu(), {k: p.grad.cpu() for k, p in params.items() if p.requires_grad}


def check_against_oracle(cfg, sd, got_loss, got, x, noise, sigma, kw, gw, simple=False, budget=None, device="cpu"):
    """Each native gradient within 8x the fp32-vs-float64 distance of the oracle's gradient (budget: of the reference's, recorded in
    tests/golden/train_meta.json, where the inputs are the fixture's: the larger of the two), plus 1e-6 relative."""
    l64, g64 = oracle_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float64, simple, device)
    l32, g32 = oracle_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float32, simple, device)
    assert torch.allclose(got_loss.double(), l64, rtol=1e-5, atol=0)
    assert set(got) == set(g64)
    for k, want in g64.items():
        zero = want == 0
        assert (got[k][zero] == 0).all(), f"{k}: nonzero where the float64 gradient is exactly zero"
        scale = want.norm().item()
        if scale == 0:
            continue
        err = (got[k].double() - want).norm().item() / scale
        ref = (g32[k].double() - want).norm().item() / scale
        if budget is not None:
            ref = max(ref, budget[k]["fp32_rel"])
        assert err <= 8 * ref + 1e-6, f"{k}: rel-L2 {err:.3e} vs the fp32 distance {ref:.3e}"


GOLDEN = Path(__file__).resolve().parent / "golden"


@pytest.mark.parametrize("simple", [False, True])
def test_class_conditional_gradients_match_float64(simple):
    cfg, inner, sd, model = build({"model": dict(CLASS["model"], loss_config="simple" if simple else "karras"), "dataset": CLASS["dataset"]})
    assert isinstance(model, K.layers.SimpleLossDenoiser) == simple
    x, noise, sigma, kw, gw = inputs(cfg, 4, 0, classes=[3, 7, 3, 1])   # class 3 in two rows, six classes in none
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw, simple)
    assert (got["class_emb.weight"][[0, 2, 4, 5, 6, 8, 9, 10]] == 0).all()


def test_three_levels_with_augment_wrapper_match_float64():
    cfg, inner, sd, model = build(LEVELS3, wrap=True)
    x, noise, sigma, kw, gw = inputs(cfg, 2, 1)
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw)


def test_odd_token_grid_and_repeated_class():
    cfg, inner, sd, model = build(CLASS)
    x, noise, sigma, kw, gw = inputs(cfg, 3, 2, size=(64, 64), classes=[5, 5, 5])
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw)


def test_two_calls_bit_identical_and_batch_is_sum_of_images():
    cfg, inner, sd, model = build(LEVELS3, wrap=True)
    x, noise, sigma, kw, gw = inputs(cfg, 3, 4)
    l1, g1 = native_grads(model, inner, x, noise, sigma, kw, gw)
    l2, g2 = native_grads(model, inner, x, noise, sigma, kw, gw)
    assert torch.equal(l1, l2) and all(torch.equal(g1[k], g2[k]) for k in g1)
    parts = [native_grads(model, inner, x[i:i + 1], noise[i:i + 1], sigma[i:i + 1], {k: v[i:i + 1] for k, v in kw.items()}, gw[i:i + 1])
             for i in range(3)]
    for k in g1:
        s = sum(p[1][k] for p in parts)
        assert (g1[k] - s).norm() <= 1e-5 * s.norm() + 1e-7, k


def test_adamw_step_on_param_groups_matches_oracle():
    cfg, inner, sd, model = build(CLASS)
    x, noise, sigma, kw, gw = inputs(cfg, 4, 5)
    _, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    _, g64 = oracle_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float64)
    lr = 2e-4
    opt = torch.optim.AdamW(inner.param_groups(lr), betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-3)
    before = {k: p.detach().clone() for k, p in inner.named_parameters()}
    opt.step()
    ref = {k: torch.nn.Parameter(v.clone().float()) for k, v in sd.items() if k in g64}
    names = {id(p): k for k, p in inner.named_parameters()}
    groups = [dict(g, params=[ref[names[id(p)]] for p in g["params"]]) for g in inner.param_groups(lr)]
    for k, p in ref.items():
        p.grad = g64[k].float()
    torch.optim.AdamW(groups, betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-3).step()
    for k, p in inner.named_parameters():
        step, want = (p.detach().cpu() - before[k].cpu()), ref[k].detach() - sd[k].float()
        assert (step - want).abs().max() <= 2e-2 * lr, k


def test_v1_training_call_is_unsupported():
    cfg = K.config.load_config({"model": {"type": "image_transformer_v1", "input_channels": 1, "input_size": [8, 8], "patch_size": [2, 2],
                                          "depth": 1, "width": 64, "d_ff": 128}})
    inner = K.config.make_model(cfg).cuda().eval()
    x = torch.randn(1, 1, 8, 8, device="cuda")
    with pytest.raises(NotImplementedError):
        K.config.make_denoiser_wrapper(cfg)(inner).loss(x, torch.randn_like(x), torch.ones(1, device="cuda"))
    eng = inner.engine()
    sig = torch.ones(1, device="cuda")
    cond = eng.conditioning(sig)
    with pytest.raises(RuntimeError, match="image_transformer_v1"):
        eng.forward_train(x, torch.randn_like(x), sig, None, None, None, cond, {})


# the reference's transformer configs: cfg1 (MNIST: d_head 64, patch 4 on a 7x7 grid, one level, no merges or splits), the CIFAR-10
# transformer (two global levels of width 256 and 512) and cfg2 (the shifted-window Oxford Flowers model, window 8 at d_head 64)
CFG1 = json.loads((GOLDEN / "cfg1_mnist_shapes.json").read_text())["config"]
CIFAR10 = json.loads((GOLDEN / "cifar10_transformer_shapes.json").read_text())["config"]
CFG2 = json.loads((GOLDEN / "cfg2_sw256_shapes.json").read_text())["config"]


@pytest.mark.parametrize("B", [2, 5])
def test_cfg1_gradients_match_float64(B):
    """cfg1 at fp32 with the cond-dropout class 10 among the labels"""
    cfg, inner, sd, model = build(CFG1)
    x, noise, sigma, kw, gw = inputs(cfg, B, 20 + B, classes=[10, 3, 10, 0, 9][:B])
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw)


@pytest.mark.parametrize("wrap", [False, True], ids=["plain", "augment_wrapper"])
def test_cifar10_transformer_gradients_match_float64(wrap):
    spec = {"model": dict(CIFAR10["model"], mapping_cond_dim=9 if wrap else 0), "dataset": CIFAR10["dataset"]}
    cfg, inner, sd, model = build(spec, wrap=wrap)
    x, noise, sigma, kw, gw = inputs(cfg, 4, 30 + wrap, classes=[10, 2, 2, 7])
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw)


def test_cifar10_transformer_batch_of_16_is_the_sum_of_its_images():
    """B = 16: level 0 holds 16 x 16 x 16 x 256 = 1,048,576 elements (TokenSplit's fac reduction loops past one pass of its grid) and
    the AdaRMSNorm scale gradients fill 16 per-image slots"""
    cfg, inner, sd, model = build(CIFAR10)
    x, noise, sigma, kw, gw = inputs(cfg, 16, 32)
    l1, g1 = native_grads(model, inner, x, noise, sigma, kw, gw)
    parts = [native_grads(model, inner, x[i:i + 1], noise[i:i + 1], sigma[i:i + 1], {k: v[i:i + 1] for k, v in kw.items()}, gw[i:i + 1])
             for i in range(16)]
    assert torch.equal(l1, torch.cat([p[0] for p in parts]))
    for k in g1:
        s = sum(p[1][k] for p in parts)
        assert (g1[k] - s).norm() <= 1e-5 * s.norm() + 1e-7, k


@pytest.mark.parametrize("size,B", [(64, 2), (128, 1)])
def test_cfg2_gradients_match_float64(size, B):
    """cfg2 with its first level at 16x16 and 32x32 tokens (window 8)"""
    cfg, inner, sd, model = build({"model": dict(CFG2["model"], input_size=[size, size]), "dataset": CFG2["dataset"]})
    x, noise, sigma, kw, gw = inputs(cfg, B, 40 + size)
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw)


@pytest.fixture(scope="module")
def no_tf32():
    """cuBLAS matmuls at full fp32 for the oracle on the GPU: under TF32 (operands rounded to 2^-11 instead of 2^-24) its fp32-vs-float64
    distance, and with it the gate, would loosen by three to four orders of magnitude"""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.mark.parametrize("name", ["cfg1", "cifar10"])
def test_reference_configs_at_the_training_batch_size(name, no_tf32):
    """train.py's default batch of 64 (config_mnist_transformer: 3136 level-0 rows; config_cifar10_transformer: 16384 and 4096): every
    gradient within 8x the oracle's fp32 distance, the oracle run on the GPU in float64 and fp32; two calls bit-identical"""
    assert not torch.backends.cuda.matmul.allow_tf32
    cfg, inner, sd, model = build({"cfg1": CFG1, "cifar10": CIFAR10}[name])
    x, noise, sigma, kw, gw = inputs(cfg, 64, 60)
    kw["class_cond"][:6] = 10   # cond-dropout rows among the labels
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw, device="cuda")
    l2, again = native_grads(model, inner, x, noise, sigma, kw, gw)
    assert torch.equal(loss, l2) and all(torch.equal(got[k], again[k]) for k in got), "two calls differ"


FROZEN = {"mapping": ("mapping.",), "class_emb": ("class_emb.",), "level": ("down_levels.0.",), "merges_splits": ("merges.", "splits.")}


@pytest.mark.parametrize("frozen", sorted(FROZEN))
def test_frozen_parameters_leave_the_other_gradients_unchanged(frozen):
    """Only parameters that require grad are bound: a frozen subset keeps grad None, and every other gradient is bit for bit that of the
    run with all parameters"""
    cfg, inner, sd, model = build(CLASS)
    x, noise, sigma, kw, gw = inputs(cfg, 3, 50, classes=[10, 4, 4])
    _, full = native_grads(model, inner, x, noise, sigma, kw, gw)
    names = [k for k, _ in inner.named_parameters() if k.startswith(FROZEN[frozen])]
    assert names
    params = dict(inner.named_parameters())
    for k in names:
        params[k].requires_grad_(False)
    inner.zero_grad(set_to_none=True)
    loss = model.loss(x.cuda(), noise.cuda(), sigma.cuda(), **{k: v.cuda() for k, v in kw.items()})
    (loss * gw.cuda()).sum().backward()
    for k, p in params.items():
        if k in names:
            assert p.grad is None, k
        else:
            assert torch.equal(p.grad.cpu(), full[k]), k


# oracle/make_golden_train.py's cases: the three-level model there has a global middle level (the reference needs natten for neighborhood)
FIXTURE_LEVELS3 = {"model": dict(LEVELS3["model"], self_attns=[LEVELS3["model"]["self_attns"][0], {"type": "global", "d_head": 16},
                                                               LEVELS3["model"]["self_attns"][2]])}
FIXTURES = {"class": (CLASS, "karras", False), "class_simple": (CLASS, "simple", False), "levels3": (FIXTURE_LEVELS3, "karras", True),
            "cfg1": (CFG1, "karras", False), "cifar10": (CIFAR10, "karras", False)}


@pytest.mark.parametrize("case", sorted(FIXTURES))
def test_fixture_cases_within_the_references_fp32_error(case):
    """The inputs recorded from the reference: each gradient within 8x the reference's own fp32 error there (or the oracle's, the larger),
    and each loss within 8x the distance of the reference's fp32 loss from its float64 loss (or 1e-6 relative)."""
    meta = json.loads((GOLDEN / "train_meta.json").read_text())["cases"][case]
    npz = np.load(GOLDEN / "train.npz")
    spec, loss_config, wrap = FIXTURES[case]
    cfg, inner, sd, model = build({"model": dict(spec["model"], loss_config=loss_config), "dataset": spec.get("dataset", {"num_classes": 0})},
                                  wrap=wrap)
    x, noise, sigma = (torch.from_numpy(npz[f"{case}_{k}"]).float() for k in ("x", "noise", "sigma"))
    kw = {}
    if cfg["dataset"]["num_classes"]:
        kw["class_cond"] = torch.tensor([3, 3])
    if cfg["model"]["mapping_cond_dim"]:   # make_golden_train draws aug_cond and mapping_cond after x, noise and sigma from one generator
        g = torch.Generator().manual_seed(11)
        for t in (x, noise, sigma):
            torch.randn(t.shape, generator=g)
        kw["aug_cond"] = torch.randn(2, 9, generator=g) * 0.3
        kw["mapping_cond"] = torch.randn(2, cfg["model"]["mapping_cond_dim"] - 9, generator=g)
    gw = torch.ones(2)   # the fixture's gradients are of loss.sum()
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    l64, l32 = (torch.from_numpy(npz[f"{case}_loss_{t}"]) for t in ("float64", "float32"))
    assert ((loss.double() - l64).abs() <= 8 * (l32 - l64).abs() + 1e-6 * l64.abs()).all(), (loss, l64, l32)
    check_against_oracle(cfg, sd, loss, got, x, noise, sigma, kw, gw, simple=loss_config == "simple", budget=meta)
