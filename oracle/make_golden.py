#!/usr/bin/env python
"""Generate tests/golden/* by running the REAL reference (imported from the checkout named by $K_DIFFUSION_REFERENCE).

Run by hand on a machine with a reference checkout (nothing else needs it):

    python oracle/make_golden.py

The reference ships no tests or golden vectors (SURVEY.md section 4), so every fixture here is an
output of the reference's own code on seeded inputs.  Seven third-party modules the reference
imports at package level are absent from this image and are stubbed exactly as SURVEY.md section 8c
describes; none of them is on the path being recorded (natten / torchsde paths are NOT recorded:
they cannot run here -> those two stay "parity unpinned").

Weights come from `k_diffusion/synth.py` (loaded by file path; recipe depends only on key/shape/seed)
so fixtures hold inputs/outputs only, never weights.
"""
import importlib.util
import json
import os
import sys
import types
from pathlib import Path

os.environ["K_DIFFUSION_USE_COMPILE"] = "0"
ROOT = Path(__file__).resolve().parents[1]
REF = Path(os.environ.get("K_DIFFUSION_REFERENCE", "k-diffusion"))     # a checkout of crowsonkb/k-diffusion
OUT = ROOT / "tests" / "golden"

import numpy as np
import torch


def _stub_missing():
    def merge(base, head):
        if isinstance(base, dict) and isinstance(head, dict):
            out = dict(base)
            for k, v in head.items():
                out[k] = merge(base[k], v) if k in base else v
            return out
        return head
    mods = {
        "jsonmerge": dict(merge=merge), "torchsde": dict(BrownianTree=None), "torchdiffeq": dict(odeint=None),
        "dctorch": {}, "dctorch.functional": {}, "skimage": {}, "skimage.transform": {},
        "clip": dict(available_models=lambda: []), "cleanfid": {}, "cleanfid.inception_torchscript": dict(InceptionV3W=None),
    }
    for name, attrs in mods.items():
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
    sys.modules["dctorch"].functional = sys.modules["dctorch.functional"]
    sys.modules["skimage"].transform = sys.modules["skimage.transform"]
    sys.modules["cleanfid"].inception_torchscript = sys.modules["cleanfid.inception_torchscript"]


def _load_synth():
    spec = importlib.util.spec_from_file_location("kdb_synth", ROOT / "k-diffusion_b200" / "k_diffusion" / "synth.py")
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def hexf(t):
    return [f"{v:08x}" for v in t.detach().float().cpu().contiguous().view(torch.int32).tolist()] if t.numel() else []


def hx(t):
    return [format(int(v) & 0xFFFFFFFF, "08x") for v in t.detach().float().cpu().contiguous().view(torch.int32).flatten().tolist()]


def main():
    _stub_missing()
    sys.path.insert(0, str(REF))
    import k_diffusion as K
    from k_diffusion.models import image_transformer_v2 as itv2
    from k_diffusion.models.axial_rope import make_axial_pos
    synth = _load_synth()
    torch.set_num_threads(8)
    OUT.mkdir(parents=True, exist_ok=True)

    # ---------------------------------------------------------------- scalar / schedule KATs
    S = K.sampling
    kat = {"schedules": [], "ancestral": [], "toy": {}, "discrete": {}, "layers": {}}
    for n, lo, hi, rho in [(10, 1e-2, 80, 7.0), (5, 1e-2, 160, 7.0), (50, 1e-2, 160, 7.0), (25, 1e-2, 160, 7.0), (1, 0.1, 10, 7.0), (7, 0.02, 14.6, 5.0)]:
        kat["schedules"].append(dict(fn="karras", args=[n, lo, hi, rho], hex=hx(S.get_sigmas_karras(n, lo, hi, rho))))
    for n, lo, hi in [(5, 1e-2, 80), (25, 1e-2, 160)]:
        kat["schedules"].append(dict(fn="exponential", args=[n, lo, hi], hex=hx(S.get_sigmas_exponential(n, lo, hi))))
    for n, lo, hi, rho in [(5, 1e-2, 80, 2.0), (12, 1e-2, 160, 1.0)]:
        kat["schedules"].append(dict(fn="polyexponential", args=[n, lo, hi, rho], hex=hx(S.get_sigmas_polyexponential(n, lo, hi, rho))))
    for n, bd, bm, es in [(5, 19.9, 0.1, 1e-3), (20, 19.9, 0.1, 1e-3)]:
        kat["schedules"].append(dict(fn="vp", args=[n, bd, bm, es], hex=hx(S.get_sigmas_vp(n, bd, bm, es))))

    sig = S.get_sigmas_karras(5, 1e-2, 80)
    for eta in (1.0, 0.5, 0.0):
        for i in range(5):
            d, u = S.get_ancestral_step(sig[i], sig[i + 1], eta=eta)
            kat["ancestral"].append(dict(eta=eta, sigma_from=hx(sig[i])[0], sigma_to=hx(sig[i + 1])[0],
                                         down=float(d), up=float(u)))

    toy = lambda x, s, **kw: 0.5 * x
    x1 = torch.ones(2, 1, 4, 4)
    for name in ("sample_euler", "sample_heun", "sample_dpmpp_2m", "sample_dpm_2", "sample_lms"):
        kat["toy"][name] = float(getattr(S, name)(toy, x1, sig, disable=True).flatten()[0])
    # nonlinear toy (sigma-dependent) exercises every coefficient path
    toy2 = lambda x, s, **kw: x / (1 + s[:, None, None, None] ** 2) + 0.1 * torch.tanh(x)
    g = torch.Generator().manual_seed(7)
    x2 = torch.randn(3, 2, 5, 5, generator=g) * 80
    sig10 = S.get_sigmas_karras(10, 1e-2, 80)
    toy_out = {}
    for name in ("sample_euler", "sample_heun", "sample_dpmpp_2m"):
        toy_out[name] = getattr(S, name)(toy2, x2, sig10, disable=True)
    noise_list = [torch.randn(3, 2, 5, 5, generator=g) for _ in range(10)]
    it = iter(noise_list)
    toy_out["sample_euler_ancestral"] = S.sample_euler_ancestral(toy2, x2, sig10, disable=True, noise_sampler=lambda a, b: next(it))
    it = iter(noise_list)
    toy_out["sample_euler_ancestral_eta05"] = S.sample_euler_ancestral(toy2, x2, sig10, disable=True, eta=0.5, s_noise=0.9, noise_sampler=lambda a, b: next(it))
    # exponential schedule without trailing zero handling differences
    np.savez(OUT / "toy_samplers.npz", x=x2.numpy(), sigmas=sig10.numpy(), noise=torch.stack(noise_list).numpy(),
             **{k: v.numpy() for k, v in toy_out.items()})

    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000) ** 2
    ac = torch.cumprod(1 - betas, 0)
    ds = K.external.DiscreteSchedule(((1 - ac) / ac) ** 0.5, True)
    q = torch.tensor([0.5, 3.3, 20.0, 0.029, 14.6, 1.0])
    kat["discrete"] = dict(
        sigma_min=float(ds.sigma_min), sigma_max=float(ds.sigma_max),
        get_sigmas_10=hx(ds.get_sigmas(10)), get_sigmas_37=hx(ds.get_sigmas(37)),
        get_sigmas_all_head=hx(ds.get_sigmas()[:5]), get_sigmas_all_tail=hx(ds.get_sigmas()[-5:]), get_sigmas_all_len=len(ds.get_sigmas()),
        roundtrip_t=ds.sigma_to_t(ds.get_sigmas(10)[:-1]).tolist(),
        query=hx(q), t_quant=ds.sigma_to_t(q).tolist(), t_interp=hx(ds.sigma_to_t(q, quantize=False)),
        t_to_sigma=hx(ds.t_to_sigma(torch.tensor([0.0, 0.5, 17.25, 998.9, 999.0]))),
    )
    den = K.Denoiser(None, sigma_data=0.5)
    cs, co, ci = den.get_scalings(torch.tensor([0.01, 0.5, 3.0, 160.0]))
    kat["scalings"] = dict(sigma_data=0.5, sigma=[0.01, 0.5, 3.0, 160.0], c_skip=hx(cs), c_out=hx(co), c_in=hx(ci))

    kat["layers"]["rope_freqs_32_2"] = hx(itv2.AxialRoPE(32, 2).freqs)
    kat["layers"]["rope_freqs_32_8"] = hx(itv2.AxialRoPE(32, 8).freqs)
    kat["layers"]["axial_pos_4_4"] = hx(make_axial_pos(4, 4))
    kat["layers"]["axial_pos_7_7"] = hx(make_axial_pos(7, 7))
    kat["layers"]["axial_pos_4_8"] = hx(make_axial_pos(4, 8))
    kat["layers"]["downscale_pos_8_8"] = hx(itv2.downscale_pos(make_axial_pos(8, 8).view(8, 8, 2)))
    m = itv2.make_shifted_window_masks(2, 3, 4, 4, 2)
    kat["layers"]["sw_mask_2_3_4_4_2"] = "".join("1" if b else "0" for b in m.flatten().tolist())
    tm = itv2.TokenMerge(1, 4, (2, 2))
    a = torch.arange(16.0).view(1, 4, 4, 1)
    from einops import rearrange
    kat["layers"]["token_merge_4x4"] = rearrange(a, "... (h nh) (w nw) e -> ... h w (nh nw e)", nh=2, nw=2).flatten().tolist()
    (OUT / "kat.json").write_text(json.dumps(kat, indent=1))

    # ---------------------------------------------------------------- model fixtures
    def build(cfg_path, overrides=None):
        cfg = json.loads((REF / "configs" / cfg_path).read_text())
        for k, v in (overrides or {}).items():
            cfg["model"][k] = v
        cfg = K.config.load_config(cfg)
        inner = K.config.make_model(cfg).eval().requires_grad_(False)
        base = inner.state_dict()
        sd = synth.synth_state_dict({k: v.shape for k, v in base.items()}, seed=1, base=base)
        inner.load_state_dict(sd)
        return cfg, inner, K.config.make_denoiser_wrapper(cfg)(inner)

    # cfg1: MNIST transformer, B=4 (BASELINE.json configs[0])
    cfg, inner, model = build("config_mnist_transformer.json")
    g = torch.Generator().manual_seed(123)
    x = torch.randn(4, 1, 28, 28, generator=g) * 80
    cc = torch.tensor([0, 1, 2, 10])
    aug = torch.randn(4, 9, generator=g) * 0.3
    sig_t = torch.tensor([0.05, 1.0, 10.0, 80.0])
    sigmas = S.get_sigmas_karras(10, 1e-2, 80)
    nz = [torch.randn(4, 1, 28, 28, generator=g) for _ in range(10)]
    with torch.no_grad():
        out = dict(
            x=x, class_cond=cc, aug_cond=aug, sigma=sig_t, sigmas=sigmas, noise=torch.stack(nz),
            inner=inner(x * 0.01, sig_t, class_cond=cc), inner_aug=inner(x * 0.01, sig_t, aug_cond=aug, class_cond=cc),
            denoised=model(x, sig_t, class_cond=cc),
            heun=S.sample_heun(model, x, sigmas, extra_args=dict(class_cond=cc), disable=True),
            dpmpp_2m=S.sample_dpmpp_2m(model, x, sigmas, extra_args=dict(class_cond=cc), disable=True),
            euler=S.sample_euler(model, x, sigmas, extra_args=dict(class_cond=cc), disable=True),
        )
        it = iter(nz)
        out["euler_ancestral"] = S.sample_euler_ancestral(model, x, sigmas, extra_args=dict(class_cond=cc), disable=True,
                                                          noise_sampler=lambda a, b: next(it))
    np.savez(OUT / "cfg1_mnist.npz", **{k: v.numpy() for k, v in out.items()})
    shapes = {k: list(v.shape) for k, v in inner.state_dict().items()}
    (OUT / "cfg1_mnist_shapes.json").write_text(json.dumps(dict(config=cfg, shapes=shapes), indent=1))
    from k_diffusion.models import flops
    with flops.flop_counter() as fc:
        inner(x[:1], sig_t[:1], class_cond=cc[:1])
    macs = {"cfg1_mnist": fc.flops}

    # shifted-window hourglass, reduced to 64x64 input (all three attention levels, shift 0 and 4)
    cfg, inner, model = build("config_oxford_flowers_shifted_window.json", dict(input_size=[64, 64]))
    g = torch.Generator().manual_seed(124)
    x = torch.randn(2, 3, 64, 64, generator=g) * 160
    sig_t = torch.tensor([0.3, 40.0])
    sigmas = S.get_sigmas_karras(6, 1e-2, 160)
    with torch.no_grad():
        out = dict(x=x, sigma=sig_t, sigmas=sigmas, inner=inner(x * 0.01, sig_t), denoised=model(x, sig_t),
                   heun=S.sample_heun(model, x, sigmas, disable=True), dpmpp_2m=S.sample_dpmpp_2m(model, x, sigmas, disable=True))
    np.savez(OUT / "sw64.npz", **{k: v.numpy() for k, v in out.items()})
    (OUT / "sw64_shapes.json").write_text(json.dumps(dict(config=cfg, shapes={k: list(v.shape) for k, v in inner.state_dict().items()}), indent=1))

    # cfg2 model at full 256x256, B=1, forward only (stored subsampled: every 4th pixel)
    cfg, inner, model = build("config_oxford_flowers_shifted_window.json")
    g = torch.Generator().manual_seed(125)
    x = torch.randn(1, 3, 256, 256, generator=g) * 160
    sig_t = torch.tensor([2.5])
    with torch.no_grad():
        with flops.flop_counter() as fc:
            o = inner(x * 0.01, sig_t)
        macs["cfg2_sw256"] = fc.flops
        d = model(x, sig_t)
    np.savez(OUT / "cfg2_sw256.npz", seed=125, sigma=sig_t.numpy(), inner_sub=o[..., ::4, ::4].numpy(), denoised_sub=d[..., ::4, ::4].numpy(),
             inner_mean=o.double().mean().item(), inner_sqmean=o.double().pow(2).mean().item())
    (OUT / "cfg2_sw256_shapes.json").write_text(json.dumps(dict(config=cfg, shapes={k: list(v.shape) for k, v in inner.state_dict().items()}), indent=1))

    # neighbourhood config: shapes/config only (natten absent -> no outputs; parity unpinned)
    cfg = K.config.load_config(json.loads((REF / "configs" / "config_oxford_flowers.json").read_text()))
    (OUT / "cfg3_na256_config.json").write_text(json.dumps(dict(config=cfg), indent=1))
    (OUT / "macs.json").write_text(json.dumps(macs, indent=1))
    print("golden written to", OUT, "MACs:", macs)


if __name__ == "__main__":
    main()
