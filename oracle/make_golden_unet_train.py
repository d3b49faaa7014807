#!/usr/bin/env python
"""The reference's training loss and parameter gradients of the image_v1 U-Net as data, recorded from the REAL reference (build container
only; the absent third-party modules stubbed as make_golden.py does):

    K_DIFFUSION_REFERENCE=<checkout> python oracle/make_golden_unet_train.py   # -> tests/golden/unet_train.npz, unet_train_meta.json

Cases: a small two-level U-Net (no augment wrapper, a 1x1 skip conv, self-attention), the mapping_cond + augment wrapper and has_variance
edge configs of tests/golden/unet_edges.json, and the reference's mnist and cifar10 configs (tests/golden/unet_configs.json) at B = 1, all
with synth.py weights (seed 3) in eval mode and dropout_rate 0.  For each: the per-sample losses of the reference's Denoiser.loss in float64 and fp32, and for
every parameter the norm of its float64 gradient, its dot product with a fixed probe and the relative L2 distance of the fp32 gradient
from the float64 one (the reference's own fp32 error); parameters the forward never reaches (grad None) are listed as such.  Also the
names in the two param_groups of each model, in the reference's order."""
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np
import torch

import make_golden as G

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"

SMALL = {"model": {"type": "image_v1", "input_channels": 3, "input_size": [16, 16], "mapping_out": 32, "depths": [1, 2], "channels": [32, 64],
                   "self_attn_depths": [False, True], "augment_wrapper": False, "sigma_data": 0.5, "dropout_rate": 0.0,
                   "loss_weighting": "soft-min-snr"}}


def cases():
    edges = json.loads((GOLDEN / "unet_edges.json").read_text())
    configs = json.loads((GOLDEN / "unet_configs.json").read_text())
    return {"small": (SMALL, 2), "mcond_aug": (edges["mcond_aug"]["config"], 2), "variance": (edges["variance"]["config"], 2),
            "mnist": (configs["mnist"]["config"], 1), "cifar10": (configs["cifar10"]["config"], 1)}


def inputs(m, B, seed=11):
    """x, noise, sigma and the conditioning of a case; shared with tests/test_unet_train_host.py"""
    g = torch.Generator().manual_seed(seed)
    H, W = m["input_size"]
    x = torch.randn(B, m["input_channels"], H, W, generator=g) * 0.5
    noise = torch.randn(x.shape, generator=g)
    sigma = torch.exp(torch.randn(B, generator=g) * 1.2 - 0.4)
    kw = {}
    if m.get("augment_wrapper", True):
        kw["aug_cond"] = torch.randn(B, 9, generator=g) * 0.3
    if m.get("mapping_cond_dim", 0):
        kw["mapping_cond"] = torch.randn(B, m["mapping_cond_dim"], generator=g)
    return x, noise, sigma, kw


def probe(shape, key):
    return torch.randn(shape, generator=torch.Generator().manual_seed(sum(map(ord, key))), dtype=torch.float64)


def main():
    G._stub_missing()
    sys.path.insert(0, str(G.REF))
    import k_diffusion as K
    synth = G._load_synth()
    torch.set_num_threads(8)
    rec, meta = {}, {"param_groups": {}, "cases": {}, "configs": {}, "no_grad": {}}
    for name, (cfg, B) in cases().items():
        c = K.config.load_config(json.loads(json.dumps(cfg)))
        # the reference's SelfAttention2d passes its dropout_p to scaled_dot_product_attention in eval mode too (layers.py:198), so the
        # recording runs without dropout, as native training does
        c["model"]["dropout_rate"] = 0.0
        model = K.config.make_model(c)
        inner = model.inner_model if isinstance(model, K.augmentation.KarrasAugmentWrapper) else model
        inner.load_state_dict(synth.synth_state_dict({k: list(v.shape) for k, v in inner.state_dict().items()}, 3, {}))
        names = {id(p): k for k, p in inner.named_parameters()}
        meta["param_groups"][name] = [[names[id(p)] for p in g["params"]] for g in inner.param_groups()]
        meta["configs"][name] = c
        x, noise, sigma, kw = inputs(c["model"], B)
        grads = {}
        for dt in (torch.float64, torch.float32):
            model = model.to(dt).eval()
            den = K.layers.Denoiser(model, c["model"]["sigma_data"], weighting=c["model"]["loss_weighting"])
            inner.zero_grad(set_to_none=True)
            loss = den.loss(x.to(dt), noise.to(dt), sigma.to(dt), **{k: v.to(dt) for k, v in kw.items()})
            loss.sum().backward()
            rec[f"{name}_loss_{str(dt)[6:]}"] = loss.detach().double().numpy()
            grads[dt] = {k: None if p.grad is None else p.grad.detach().double() for k, p in inner.named_parameters()}
        case = {}
        for k, g64 in grads[torch.float64].items():
            if g64 is None:
                continue
            n = g64.norm().item()
            case[k] = dict(norm=n, probe=(g64 * probe(g64.shape, k)).sum().item(),
                           fp32_rel=(grads[torch.float32][k] - g64).norm().item() / n if n > 0 else 0.0)
        meta["cases"][name] = case
        meta["no_grad"][name] = sorted(k for k, g in grads[torch.float64].items() if g is None)
        for k, v in dict(x=x, noise=noise, sigma=sigma, **kw).items():
            rec[f"{name}_{k}"] = v.numpy()
    np.savez_compressed(GOLDEN / "unet_train.npz", **rec)
    (GOLDEN / "unet_train_meta.json").write_text(json.dumps(meta, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
