#!/usr/bin/env python
"""Generate tests/golden/unet_*.{json,npz} by running the REAL reference image_v1 U-Net (checkout named by $K_DIFFUSION_REFERENCE).

Run by hand on a machine with a reference checkout (nothing else needs it):

    python oracle/make_golden_unet.py

For each of the reference's four image_v1 configs it records the merged config, the state-dict keys and shapes of
config.make_model (KarrasAugmentWrapper(ImageDenoiserModelV1)), and Denoiser outputs on seeded inputs with the synth
weights (k_diffusion/synth.py: zero-initialised tensors re-randomised) and eval semantics: the reference's
SelfAttention2d passes its dropout rate to scaled_dot_product_attention whatever the module's mode (layers.py:198), so
every nn.Dropout's p is set to 0 to record the deterministic function a sampler is meant to evaluate.  B = 3 at sigma = sigma_min, 1, sigma_max (one per
image), without and with a nonzero aug_cond.  config_mnist also gets one Heun-10 trajectory.  Weights are never stored.
"""
import json
import sys
from pathlib import Path

import numpy as np
import torch

from make_golden import OUT, REF, _load_synth, _stub_missing

CONFIGS = {"mnist": "config_mnist.json", "cifar10": "config_cifar10.json", "32x32_small": "config_32x32_small.json",
           "32x32_small_butterflies": "config_32x32_small_butterflies.json"}
EDGE_BASE = "config_cifar10.json"
EDGES = {
    "odd_nonsquare": dict(input_size=[20, 36], depths=[1, 2, 1], channels=[36, 68, 96], self_attn_depths=[False, True, True], mapping_out=72),
    "patch2_skip1": dict(input_size=[24, 16], depths=[1, 1, 1], channels=[32, 64, 64], self_attn_depths=[False, False, True], mapping_out=64,
                         patch_size=2, skip_stages=1),
    "mcond_aug": dict(input_size=[12, 20], depths=[1, 1], channels=[32, 64], self_attn_depths=[False, True], mapping_out=64, mapping_cond_dim=5),
    "mcond_plain": dict(input_size=[12, 20], depths=[1, 1], channels=[32, 64], self_attn_depths=[False, True], mapping_out=64, mapping_cond_dim=5,
                        augment_wrapper=False),
    "identity_concat": dict(input_size=[16, 16], depths=[1, 1, 1], channels=[64, 32, 32], self_attn_depths=[False, False, False], mapping_out=64),
    "variance": dict(input_size=[8, 8], depths=[1, 1], channels=[32, 64], self_attn_depths=[False, False], mapping_out=64, has_variance=True),
}


def call_variants(mcfg):
    """{output key: (pass aug_cond, pass mapping_cond)} for every way the config's Denoiser can be called"""
    wrap, mc = mcfg["augment_wrapper"], mcfg["mapping_cond_dim"] > 0
    if wrap:
        return {"denoised_mc": (False, True), "denoised_aug_mc": (True, True)} if mc else {"denoised": (False, False), "denoised_aug": (True, False)}
    return {"denoised": (False, False), "denoised_mc": (False, True)} if mc else {"denoised": (False, False)}


def record(K, synth, cfg, seed):
    """(Denoiser, outputs on seeded inputs, state-dict shapes, the input generator) of a merged config with the synth weights and
    dropout p = 0"""
    model = K.config.make_model(cfg).eval().requires_grad_(False)
    for mod in model.modules():             # SelfAttention2d hands dropout.p to SDPA even in eval mode (layers.py:198)
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    base = model.state_dict()
    shapes = {k: list(v.shape) for k, v in base.items()}
    model.load_state_dict(synth.synth_state_dict({k: v.shape for k, v in base.items()}, seed=1, base=base))
    den = K.config.make_denoiser_wrapper(cfg)(model)
    m = cfg["model"]
    c, (h, w) = m["input_channels"], m["input_size"]
    g = torch.Generator().manual_seed(seed)
    sigma = torch.tensor([m["sigma_min"], 1.0, m["sigma_max"]], dtype=torch.float32)
    x = torch.randn(3, c, h, w, generator=g) * sigma[:, None, None, None] + 0.5 * torch.randn(3, c, h, w, generator=g)
    aug = torch.randn(3, 9, generator=g) * 0.5
    out = dict(x=x, sigma=sigma, aug_cond=aug)
    if m["mapping_cond_dim"] > 0:
        out["mapping_cond"] = torch.randn(3, m["mapping_cond_dim"], generator=g)
    with torch.no_grad():
        for key, (use_aug, use_mc) in call_variants(m).items():
            kw = dict(aug_cond=aug) if use_aug else {}
            if use_mc:
                kw["mapping_cond"] = out["mapping_cond"]
            out[key] = den(x, sigma, **kw)
    return den, out, shapes, g


def main():
    _stub_missing()
    sys.path.insert(0, str(REF))
    import k_diffusion as K
    synth = _load_synth()
    torch.set_num_threads(8)
    meta = {}
    for seed, (name, path) in enumerate(CONFIGS.items()):
        cfg = K.config.load_config(json.loads((REF / "configs" / path).read_text()))
        den, out, shapes, g = record(K, synth, cfg, 200 + seed)
        m = cfg["model"]
        c, (h, w) = m["input_channels"], m["input_size"]
        with torch.no_grad():
            if name == "mnist":
                xt = torch.randn(2, c, h, w, generator=g) * m["sigma_max"]
                sigmas = K.sampling.get_sigmas_karras(10, m["sigma_min"], m["sigma_max"])
                out.update(heun_x=xt, heun_sigmas=sigmas, heun=K.sampling.sample_heun(den, xt, sigmas, disable=True))
        np.savez_compressed(OUT / f"unet_{name}.npz", **{k: v.numpy() for k, v in out.items()})
        meta[name] = dict(config=cfg, shapes=shapes)
    (OUT / "unet_configs.json").write_text(json.dumps(meta, indent=1))
    edges = {}
    for seed, (name, over) in enumerate(EDGES.items()):
        cfg = json.loads((REF / "configs" / EDGE_BASE).read_text())
        cfg["model"].update(over)
        cfg = K.config.load_config(cfg)
        _, out, shapes, _ = record(K, synth, cfg, 300 + seed)
        np.savez_compressed(OUT / f"unet_edge_{name}.npz", **{k: v.numpy() for k, v in out.items()})
        edges[name] = dict(config=cfg, shapes=shapes)
    (OUT / "unet_edges.json").write_text(json.dumps(edges, indent=1))
    print("golden written to", OUT)


if __name__ == "__main__":
    main()
