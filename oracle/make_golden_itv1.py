#!/usr/bin/env python
"""Generate tests/golden/itv1_*.{json,npz} by running the REAL reference image_transformer_v1 (checkout named by $K_DIFFUSION_REFERENCE).

Run by hand on a machine with a reference checkout (nothing else needs it):

    python oracle/make_golden_itv1.py

The reference ships no image_transformer_v1 config, so three are defined here: an MNIST-sized class-conditional one, a CIFAR-sized
one and an edge case with a non-square image and a non-square patch (which pins the aspect-ratio rule of the positions).  For each it
records the merged config, the state-dict keys and shapes of config.make_model, and Denoiser outputs with the synth weights
(k_diffusion/synth.py) at sigma = sigma_min, 1, sigma_max (one per image), without and with a nonzero aug_cond, per-sample class_cond
where the config has classes, and the raw inner model.  The MNIST-sized config also gets one Heun-10 trajectory, and every config the
reference's own distance between its fp32 forward and its forward under autocast(bfloat16) (the bf16 budget).  The constructor and
forward signatures go to itv1_meta.json.  Weights are never stored.
"""
import inspect
import json
import sys

import numpy as np
import torch

from make_golden import OUT, REF, _load_synth, _stub_missing

BASE = {"model": {"type": "image_transformer_v1", "sigma_data": 1.0, "sigma_min": 1e-2, "sigma_max": 80.0}, "dataset": {"num_classes": 0}}
CONFIGS = {
    "mnist": dict(model=dict(input_channels=1, input_size=[28, 28], patch_size=[2, 2], width=256, depth=4), num_classes=10),
    "cifar": dict(model=dict(input_channels=3, input_size=[32, 32], patch_size=[2, 2], width=512, depth=8, sigma_max=160.0), num_classes=0),
    "edge": dict(model=dict(input_channels=3, input_size=[24, 40], patch_size=[2, 4], width=128, depth=2), num_classes=0),
}


def config(name):
    c = json.loads(json.dumps(BASE))
    c["model"].update(CONFIGS[name]["model"])
    c["dataset"]["num_classes"] = CONFIGS[name]["num_classes"]
    return c


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def main():
    _stub_missing()
    sys.path.insert(0, str(REF))
    import k_diffusion as K
    synth = _load_synth()
    torch.set_num_threads(8)
    meta = {"api": {"__init__": str(inspect.signature(K.models.ImageTransformerDenoiserModelV1.__init__)),
                    "forward": str(inspect.signature(K.models.ImageTransformerDenoiserModelV1.forward))}, "configs": {}}
    for seed, name in enumerate(CONFIGS):
        cfg = K.config.load_config(config(name))
        model = K.config.make_model(cfg).eval().requires_grad_(False)
        base = model.state_dict()
        shapes = {k: list(v.shape) for k, v in base.items()}
        model.load_state_dict(synth.synth_state_dict({k: v.shape for k, v in base.items()}, seed=1, base=base))
        den = K.config.make_denoiser_wrapper(cfg)(model)
        m = cfg["model"]
        c, (h, w) = m["input_channels"], m["input_size"]
        g = torch.Generator().manual_seed(400 + seed)
        sigma = torch.tensor([m["sigma_min"], 1.0, m["sigma_max"]], dtype=torch.float32)
        x = torch.randn(3, c, h, w, generator=g) * sigma[:, None, None, None] + 0.5 * torch.randn(3, c, h, w, generator=g)
        aug = torch.randn(3, 9, generator=g) * 0.5
        out = dict(x=x, sigma=sigma, aug_cond=aug)
        kw = {}
        if cfg["dataset"]["num_classes"]:
            out["class_cond"] = kw["class_cond"] = torch.tensor([0, 7, cfg["dataset"]["num_classes"]])   # the last: the CFG token
        with torch.no_grad():
            out["denoised"] = den(x, sigma, **kw)
            out["denoised_aug"] = den(x, sigma, aug_cond=aug, **kw)
            out["inner"] = model(x, sigma, **kw)
            with torch.autocast("cpu", dtype=torch.bfloat16):
                bf = den(x, sigma, **kw).float()
            budget = {"forward_rel_l2": rel_l2(bf, out["denoised"])}
            if name == "mnist":
                xt = torch.randn(2, c, h, w, generator=g) * m["sigma_max"]
                sigmas = K.sampling.get_sigmas_karras(10, m["sigma_min"], m["sigma_max"])
                cc = torch.tensor([3, 10])
                out.update(heun_x=xt, heun_sigmas=sigmas, heun_class_cond=cc,
                           heun=K.sampling.sample_heun(den, xt, sigmas, extra_args=dict(class_cond=cc), disable=True))
                with torch.autocast("cpu", dtype=torch.bfloat16):
                    hb = K.sampling.sample_heun(den, xt, sigmas, extra_args=dict(class_cond=cc), disable=True).float()
                budget["heun10_rel_l2"] = rel_l2(hb, out["heun"])
        np.savez_compressed(OUT / f"itv1_{name}.npz", **{k: v.numpy() for k, v in out.items()})
        meta["configs"][name] = dict(config=cfg, shapes=shapes, bf16_budget=budget)
    (OUT / "itv1_meta.json").write_text(json.dumps(meta, indent=1))
    print("golden written to", OUT)


if __name__ == "__main__":
    main()
