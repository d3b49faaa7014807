"""The reference's training loop on the H100: sigma sample densities on CUDA against the oracle's restatement, ema_update through
kdb_ema_update against per-tensor lerp_ / copy_ bit for bit, the EMA model's engine rebinding after the update, and 20 steps in the shape of
train.py's loop side by side with the oracle under torch autograd."""
import copy
import json

import pytest
import torch

from conftest import GOLDEN, synth_sd
from oracle import kdiff_oracle as O
from oracle import train_loop_oracle as TO

import k_diffusion as K

pytestmark = pytest.mark.gpu

META = json.loads((GOLDEN / "train_loop.json").read_text())


def test_densities_on_cuda_equal_the_oracle_bit_for_bit():
    for case, cfg in sorted(META["densities"].items()):
        density = K.config.make_sample_density(cfg)
        for i, strat in enumerate(META["strats"]):
            torch.manual_seed(2000 + i)
            if strat is None:
                got = density([1000], device="cuda")
            else:
                with K.utils.enable_stratified(*strat):
                    got = density([1000], device="cuda")
            torch.manual_seed(2000 + i)
            want = TO.sample_density(cfg, [1000], "cuda", strat)
            assert got.is_cuda and got.dtype == want.dtype and torch.equal(got, want), (case, strat)


def _cfg(stem):
    return json.loads((GOLDEN / f"{stem}_shapes.json").read_text())["config"]


def _transformer(stem, seed):
    cfg = K.config.load_config(_cfg(stem))
    model = K.config.make_model(cfg)
    model.load_state_dict(synth_sd({k: list(v.shape) for k, v in model.state_dict().items()}, seed))
    return model


def _unet(seed):
    cfg = K.config.load_config(json.loads((GOLDEN / "unet_configs.json").read_text())["cifar10"]["config"])
    model = K.config.make_model(cfg)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for t in model.state_dict().values():
            if t.is_floating_point():
                t.copy_(torch.randn(t.shape, generator=g) * 0.1)
    return model


class Edge(torch.nn.Module):
    """Parameters of 0, 1, 3 and 4k + 1 elements, two views into a shared storage starting `shift` + 1 and `shift` + 2 floats in (made on
    `device`: moving a view copies it to a fresh storage) and a buffer."""

    def __init__(self, seed, shift, device="cuda"):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        for i, n in enumerate((0, 1, 3, 4 * 1000 + 1, 4 * 12345 + 1)):
            setattr(self, f"p{i}", torch.nn.Parameter(torch.randn(n, generator=g).to(device)))
        base = torch.randn(10000, generator=g).to(device)
        self.v0 = torch.nn.Parameter(base[1 + shift:4002 + shift])
        self.v1 = torch.nn.Parameter(base[4006 + shift:9003 + shift])
        self.register_buffer("running", torch.randn(77, generator=g).to(device))


MODELS = {"cfg1": lambda s: _transformer("cfg1_mnist", s).cuda(), "cfg2": lambda s: _transformer("cfg2_sw256", s).cuda(),
          "unet_cifar10": lambda s: _unet(s).cuda(), "edge_aligned": lambda s: Edge(s, 0), "edge_misaligned": lambda s: Edge(s, s)}


def _per_tensor(model, ema, decay):
    """the reference's ema_update (utils.py:88-104)"""
    with torch.no_grad():
        pe = dict(ema.named_parameters())
        for k, p in model.named_parameters():
            pe[k].lerp_(p, 1 - decay)
        be = dict(ema.named_buffers())
        for k, b in model.named_buffers():
            be[k].copy_(b)


@pytest.mark.parametrize("name", sorted(MODELS))
@pytest.mark.parametrize("decay", [0., 0.5, 0.999, 1.])
def test_ema_update_is_bit_identical_to_per_tensor_lerp(name, decay):
    model, ema = MODELS[name](1), MODELS[name](2)
    if name.startswith("edge"):   # aligned: the views of both sit alike off a 16-byte boundary; misaligned: 4 bytes apart
        assert (ema.v0.data_ptr() - model.v0.data_ptr()) % 16 == (0 if name == "edge_aligned" else 4)
        assert ema.v0.data_ptr() % 16 != 0
    want = copy.deepcopy(ema)
    _per_tensor(model, want, decay)
    before = K._native.launch_breakdown().get("ema", 0)
    K.utils.ema_update(model, ema, decay)
    assert K._native.launch_breakdown()["ema"] == before + 1   # every tensor in one launch
    got_sd, want_sd = ema.state_dict(), want.state_dict()
    for k, w in want_sd.items():
        assert torch.equal(got_sd[k].view(torch.int32) if w.dtype == torch.float32 else got_sd[k],
                           w.view(torch.int32) if w.dtype == torch.float32 else w), k


def test_lerp_branches_and_special_values_match_torch():
    g = torch.Generator().manual_seed(3)
    n = 1 << 20
    src = torch.cat([torch.randn(n, generator=g) * 10 ** torch.randint(-30, 30, (n,), generator=g).float(),
                     torch.tensor([0., -0., float("inf"), -float("inf"), float("nan"), 1e-45, 3.4e38])]).cuda()
    for decay in (0., 1e-7, 0.25, 0.5, 0.5000001, 0.75, 0.9999, 1., 1.5, -0.5):
        dst = torch.randn(src.shape, generator=g).cuda()
        want = dst.clone().lerp_(src, 1 - decay)
        K._native.ema_update([dst], [src], [K._native.EMA_LERP], 1 - decay)
        assert torch.equal(dst.view(torch.int32), want.view(torch.int32)), decay


def test_fallbacks_and_key_mismatch():
    model, ema = MODELS["edge_aligned"](1), MODELS["edge_aligned"](2)
    before = K._native.launch_breakdown().get("ema", 0)
    bf = copy.deepcopy(ema).to(torch.bfloat16)          # bf16 EMA parameters: per-tensor lerp_
    want = copy.deepcopy(bf)
    _per_tensor(model.to(torch.bfloat16), want, 0.9)
    K.utils.ema_update(model, bf, 0.9)
    assert all(torch.equal(a, b) for a, b in zip(bf.state_dict().values(), want.state_dict().values()))
    model, ema = MODELS["edge_aligned"](1), MODELS["edge_aligned"](2)
    for m, seed in ((model, 1), (ema, 2)):                # an integer buffer: per-tensor lerp_ / copy_
        m.register_buffer("count", torch.tensor(seed, device="cuda"))
    want = copy.deepcopy(ema)
    _per_tensor(model, want, 0.9)
    K.utils.ema_update(model, ema, 0.9)
    assert all(torch.equal(a, b) for a, b in zip(ema.state_dict().values(), want.state_dict().values())) and int(ema.count) == 1
    model = MODELS["edge_aligned"](1)
    cpu_ema = Edge(2, 0, "cpu")                          # mixed devices: per-tensor lerp_, which raises as the reference's does
    with pytest.raises(RuntimeError):
        K.utils.ema_update(model, cpu_ema, 0.9)
    t = torch.nn.Module()
    t.w = torch.nn.Parameter(torch.randn(8, 8, device="cuda").t())   # not contiguous: per-tensor lerp_
    e = torch.nn.Module()
    e.w = torch.nn.Parameter(torch.randn(8, 8, device="cuda"))
    w = e.w.detach().clone().lerp_(t.w.detach(), 0.25)
    K.utils.ema_update(t, e, 0.75)
    assert torch.equal(e.w.detach(), w)
    assert K._native.launch_breakdown().get("ema", 0) == before
    with pytest.raises(AssertionError):
        K.utils.ema_update(torch.nn.Linear(2, 2).cuda(), torch.nn.Sequential(torch.nn.Linear(2, 2)).cuda(), 0.9)


def test_ema_models_engine_serves_the_updated_weights():
    """kdb_ema_update writes through raw pointers; ema_update bumps each destination's version so the EMA model's engine rebinds."""
    cfg = K.config.load_config(_cfg("cfg1_mnist"))
    inner, inner_ema = _transformer("cfg1_mnist", 1).cuda().eval(), _transformer("cfg1_mnist", 2).cuda().eval()
    wrap = K.config.make_denoiser_wrapper(cfg)
    ema = wrap(inner_ema)
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(2, 1, 28, 28, generator=g) * 80).cuda()
    extra = dict(class_cond=torch.tensor([3, 10], device="cuda"))
    sigmas = K.sampling.get_sigmas_karras(4, 1e-2, 80, device="cuda")
    first = K.sampling.sample_euler(ema, x, sigmas, extra_args=extra, disable=True)
    K.utils.ema_update(inner, inner_ema, 0.5)
    second = K.sampling.sample_euler(ema, x, sigmas, extra_args=extra, disable=True)
    fresh = _transformer("cfg1_mnist", 3)
    fresh.load_state_dict(inner_ema.state_dict())
    want = K.sampling.sample_euler(wrap(fresh.cuda().eval()), x, sigmas, extra_args=extra, disable=True)
    assert torch.equal(second, want)
    assert not torch.equal(first, second)


# ---------------------------------------------------------------------------------------------
# 20 steps of train.py's loop (train.py:440-472) on cfg1, native and on the oracle
# ---------------------------------------------------------------------------------------------

STEPS, B = 20, 8
NO_GRAD = ("pos_emb.freqs", "time_emb.weight", "aug_emb.weight")


def _loop_setup():
    raw = _cfg("cfg1_mnist")
    cfg = K.config.load_config(dict(raw, model=dict(raw["model"], dropout_rate=[0.0])))   # the native training path refuses dropout
    shapes = {k: list(v.shape) for k, v in K.config.make_model(cfg).state_dict().items()}
    g = torch.Generator().manual_seed(7)
    reals = [(torch.rand(B, 1, 28, 28, generator=g) * 2 - 1) for _ in range(STEPS)]
    labels = [torch.randint(0, 10, (B,), generator=g) for _ in range(STEPS)]
    return cfg, synth_sd(shapes, 1), reals, labels


def _step_inputs(cfg, density, step, reals, labels):
    """train.py's draws for one step, from torch's CUDA generator: class dropout, noise, stratified sigmas"""
    torch.manual_seed(100 + step)
    x = reals[step].cuda()
    class_cond = labels[step].cuda()
    drop = torch.rand(class_cond.shape, device="cuda")
    class_cond.masked_fill_(drop < cfg["dataset"]["cond_dropout_rate"], cfg["dataset"]["num_classes"])
    noise = torch.randn_like(x)
    with K.utils.enable_stratified(step % 4, 4):
        sigma = density([B], device="cuda")
    return x, noise, sigma, class_cond


def _schedules(opt):
    return K.utils.InverseLR(opt, inv_gamma=50., power=0.75, warmup=0.9), K.utils.EMAWarmup(power=0.6667, max_value=0.9999)


def _native_loop(cfg, sd, reals, labels):
    inner = K.config.make_model(cfg)
    inner.load_state_dict(sd)
    inner = inner.cuda().eval()
    inner_ema = copy.deepcopy(inner)
    model = K.config.make_denoiser_wrapper(cfg)(inner)
    o = cfg["optimizer"]
    opt = torch.optim.AdamW(inner.param_groups(o["lr"]), betas=o["betas"], eps=o["eps"], weight_decay=o["weight_decay"])
    sched, ema_sched = _schedules(opt)
    density = K.config.make_sample_density(cfg["model"])
    launches = K._native.launch_breakdown().get("ema", 0)
    losses = []
    for step in range(STEPS):
        x, noise, sigma, class_cond = _step_inputs(cfg, density, step, reals, labels)
        loss = model.loss(x, noise, sigma, class_cond=class_cond)
        loss.mean().backward()
        torch.nn.utils.clip_grad_norm_(inner.parameters(), 1.)
        opt.step()
        sched.step()
        opt.zero_grad()
        K.utils.ema_update(inner, inner_ema, ema_sched.get_value())
        ema_sched.step()
        losses.append(loss.detach().double().cpu())
    assert K._native.launch_breakdown()["ema"] == launches + STEPS
    return torch.stack(losses), {k: v.detach().double().cpu() for k, v in inner_ema.state_dict().items()}


def _oracle_loop(cfg, sd, reals, labels, dtype, groups_of):
    m = cfg["model"]
    params = {k: v.to(dtype).requires_grad_(not k.endswith(NO_GRAD)) for k, v in sd.items()}   # the oracle runs on the CPU
    ema = {k: v.detach().clone() for k, v in params.items()}
    o = cfg["optimizer"]
    opt = torch.optim.AdamW([dict(g, params=[params[k] for k in keys]) for g, keys in groups_of], betas=o["betas"], eps=o["eps"],
                            weight_decay=o["weight_decay"])
    sched, ema_sched = _schedules(opt)
    density = K.config.make_sample_density(m)
    sdata = m["sigma_data"]
    losses = []
    for step in range(STEPS):
        x, noise, sigma, class_cond = _step_inputs(cfg, density, step, reals, labels)
        x, noise, sigma, class_cond = x.cpu().to(dtype), noise.cpu().to(dtype), sigma.cpu().to(dtype), class_cond.cpu()
        c_skip, c_out, c_in = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sigma, sdata)]
        noised = x + noise * sigma.view(-1, 1, 1, 1)
        f = O.model_forward(params, m, noised * c_in, sigma, class_cond=class_cond)
        w = (sigma * sdata) ** 2 / (sigma ** 2 + sdata ** 2) ** 2     # soft-min-snr (layers.py:18-19)
        loss = ((f - (x - c_skip * noised) / c_out) ** 2).flatten(1).mean(1) * w
        loss.mean().backward()
        trained = [p for p in params.values() if p.requires_grad]
        torch.nn.utils.clip_grad_norm_(trained, 1.)
        opt.step()
        sched.step()
        opt.zero_grad()
        decay = ema_sched.get_value()
        with torch.no_grad():
            for k, p in params.items():
                if p.requires_grad:
                    ema[k].lerp_(p, 1 - decay)
                else:
                    ema[k].copy_(p)
        ema_sched.step()
        losses.append(loss.detach().double().cpu())
    return torch.stack(losses), {k: v.double().cpu() for k, v in ema.items()}


def test_twenty_steps_of_train_py_match_the_oracle():
    """Per-step losses and the final EMA weights of the native loop within 8x the oracle's own fp32-vs-float64 distance (plus 1e-6
    relative), the bound tests/test_gpu_train.py puts on one step's gradients, here measured after the same steps."""
    cfg, sd, reals, labels = _loop_setup()
    inner = K.config.make_model(cfg)
    names = {id(p): k for k, p in inner.named_parameters()}
    groups_of = [({k: v for k, v in g.items() if k != "params"}, [names[id(p)] for p in g["params"]])
                 for g in inner.param_groups(cfg["optimizer"]["lr"])]
    l_nat, e_nat = _native_loop(cfg, sd, reals, labels)
    l64, e64 = _oracle_loop(cfg, sd, reals, labels, torch.float64, groups_of)
    l32, e32 = _oracle_loop(cfg, sd, reals, labels, torch.float32, groups_of)
    for s in range(STEPS):
        err = (l_nat[s] - l64[s]).norm() / l64[s].norm()
        ref = (l32[s] - l64[s]).norm() / l64[s].norm()
        assert err <= 8 * ref + 1e-6, f"step {s}: loss rel-L2 {err:.3e} vs the oracle's fp32 distance {ref:.3e}"
    assert set(e_nat) == set(e64)
    moved = 0
    for k, want in e64.items():
        scale = want.norm()
        if scale == 0:
            assert (e_nat[k] == 0).all(), k
            continue
        err = (e_nat[k] - want).norm() / scale
        ref = (e32[k] - want).norm() / scale
        assert err <= 8 * ref + 1e-6, f"{k}: EMA rel-L2 {err:.3e} vs the oracle's fp32 distance {ref:.3e}"
        moved += not torch.equal(e64[k], sd[k].double())
    assert moved > 0
