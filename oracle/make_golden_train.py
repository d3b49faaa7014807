#!/usr/bin/env python
"""The reference's training loss and parameter gradients of image_transformer_v2 as data, recorded from the REAL reference (build container
only; natten, dctorch and the other absent modules stubbed):

    K_DIFFUSION_REFERENCE=<checkout> python oracle/make_golden_train.py      # -> tests/golden/train.npz, tests/golden/train_meta.json

For a class-conditional model (soft-min-snr, and the simple loss), a three-level model (shifted-window, global and none levels,
mapping_cond, aug_cond through KarrasAugmentWrapper), cfg1 (the MNIST transformer) and the CIFAR-10 transformer, with synth.py weights: the per-sample losses of Denoiser.loss in float64 and fp32,
and for every parameter the norm of its float64 gradient, its dot product with a fixed probe, and the relative L2 distance of the fp32
gradient from the float64 one (the reference's own fp32 error).  Also the names of the four param_groups of those models and of cfg1.
The inputs follow tests/test_train_host.py's recipe."""
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np
import torch

import make_golden as G
from oracle import kdiff_oracle as O

ROOT = Path(__file__).resolve().parents[1]

CLASS = {"model": {"type": "image_transformer_v2", "input_channels": 1, "input_size": [16, 16], "patch_size": [2, 2], "depths": [2, 1],
                   "widths": [32, 64], "d_ffs": [64, 96], "mapping_width": 64, "mapping_depth": 2, "mapping_d_ff": 96,
                   "loss_weighting": "soft-min-snr", "sigma_data": 0.6,
                   "self_attns": [{"type": "shifted-window", "d_head": 16, "window_size": 4}, {"type": "global", "d_head": 16}]},
         "dataset": {"num_classes": 10}}
LEVELS3 = {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [32, 32], "patch_size": [2, 2], "depths": [1, 1, 1],
                     "widths": [32, 48, 64], "d_ffs": [64, 96, 128], "mapping_width": 64, "mapping_depth": 1, "mapping_d_ff": 128,
                     "mapping_cond_dim": 12, "sigma_data": 0.5,
                     "self_attns": [{"type": "shifted-window", "d_head": 16, "window_size": 4}, {"type": "global", "d_head": 16},
                                    {"type": "none"}]}}
CASES = {"class": (CLASS, "karras", False), "class_simple": (CLASS, "simple", False), "levels3": (LEVELS3, "karras", True)}
# the reference's own transformer configs: cfg1 (MNIST, tests/golden/cfg1_mnist_shapes.json) and the CIFAR-10 transformer, whose loaded
# config and parameter shapes this script records in tests/golden/cifar10_transformer_shapes.json
REF_CASES = {"cfg1": "cfg1_mnist_shapes.json", "cifar10": "cifar10_transformer_shapes.json"}


def synth_sd(synth, shapes, seed=3):
    base = {k: O.rope_freqs(s[1] * 8, s[0]) for k, s in shapes.items() if k.endswith("pos_emb.freqs")}
    return synth.synth_state_dict(shapes, seed, base)


def inputs(m, num_classes, B=2, seed=11):
    g = torch.Generator().manual_seed(seed)
    H, W = m["input_size"]
    x = torch.randn(B, m["input_channels"], H, W, generator=g) * 0.5
    noise = torch.randn(x.shape, generator=g)
    sigma = torch.exp(torch.randn(B, generator=g) * 1.2 - 0.4)
    kw = {}
    if num_classes:
        kw["class_cond"] = torch.tensor([3, 3][:B])
    if m.get("mapping_cond_dim", 0):
        kw["aug_cond"] = torch.randn(B, 9, generator=g) * 0.3
        kw["mapping_cond"] = torch.randn(B, m["mapping_cond_dim"] - 9, generator=g)
    return x, noise, sigma, kw


def probe(shape, key):
    return torch.randn(shape, generator=torch.Generator().manual_seed(sum(map(ord, key))), dtype=torch.float64)


def names_of(model, groups):
    names = {id(p): k for k, p in model.named_parameters()}
    return [[names[id(p)] for p in g["params"]] for g in groups]


def main():
    G._stub_missing()
    sys.path.insert(0, str(G.REF))
    import k_diffusion as K
    synth = G._load_synth()
    torch.set_num_threads(8)
    rec, meta = {}, {"param_groups": {}, "cases": {}}
    golden = ROOT / "tests" / "golden"
    c10 = K.config.load_config(json.loads((G.REF / "configs" / "config_cifar10_transformer.json").read_text()))
    shapes = {k: list(v.shape) for k, v in K.config.make_model(c10).state_dict().items()}
    (golden / REF_CASES["cifar10"]).write_text(json.dumps(dict(config=c10, shapes=shapes), indent=1))
    cases = dict(CASES, **{name: (json.loads((golden / f).read_text())["config"], "karras", False) for name, f in REF_CASES.items()})
    for name, (cfg, loss_config, wrap) in cases.items():
        c = K.config.load_config(json.loads(json.dumps(cfg)))
        c["model"]["loss_config"] = loss_config
        inner = K.config.make_model(c)
        sd = synth_sd(synth, {k: list(v.shape) for k, v in inner.state_dict().items()})
        inner.load_state_dict(sd)
        meta["param_groups"][name] = names_of(inner, inner.param_groups())
        x, noise, sigma, kw = inputs(c["model"], c["dataset"]["num_classes"])
        grads = {}
        for dt in (torch.float64, torch.float32):
            inner = inner.to(dt).eval()
            model = K.config.make_denoiser_wrapper(c)(K.augmentation.KarrasAugmentWrapper(inner) if wrap else inner)
            inner.zero_grad(set_to_none=True)
            kwd = {k: (v.to(dt) if v.is_floating_point() else v) for k, v in kw.items()}
            loss = model.loss(x.to(dt), noise.to(dt), sigma.to(dt), **kwd)
            loss.sum().backward()
            rec[f"{name}_loss_{str(dt)[6:]}"] = loss.detach().double().numpy()
            grads[dt] = {k: p.grad.detach().double() for k, p in inner.named_parameters()}
        case = {}
        for k, g64 in grads[torch.float64].items():
            n = g64.norm().item()
            case[k] = dict(norm=n, probe=(g64 * probe(g64.shape, k)).sum().item(),
                           fp32_rel=(grads[torch.float32][k] - g64).norm().item() / n if n > 0 else 0.0)
        meta["cases"][name] = case
        for k in ("x", "noise", "sigma"):
            rec[f"{name}_{k}"] = locals()[k].numpy()
    c1 = json.loads((ROOT / "tests" / "golden" / "cfg1_mnist_shapes.json").read_text())["config"]
    cfg1 = K.config.load_config(c1)
    m1 = K.config.make_model(cfg1)
    meta["param_groups"]["cfg1"] = names_of(m1, m1.param_groups())
    out = ROOT / "tests" / "golden"
    np.savez_compressed(out / "train.npz", **rec)
    (out / "train_meta.json").write_text(json.dumps(meta, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
