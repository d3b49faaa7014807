#!/usr/bin/env python
"""Golden outputs of the reference's classifier-free-guidance closure (build container only):

    python oracle/make_golden_cfg.py        # -> tests/golden/cfg1_cfg.npz

`make_cfg_model_fn` is a closure inside train.py's main() (train.py:333-344) and cannot be imported, so this script cuts its
source lines out of the reference's train.py ($K_DIFFUSION_REFERENCE) AT RUN TIME (nothing is copied into the repo) and executes them with the two
free variables it reads (`cfg_scale`, `num_classes`) bound.  The recorded run is the reference's own demo() recipe
(train.py:363: sample_dpmpp_2m_sde, eta=0, solver_type='heun') on the cfg1 MNIST model (10 classes + unconditional token)."""
import json
import sys
import textwrap
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
import numpy as np
import torch

import make_golden as G


def reference_closure(cfg_scale, num_classes):
    lines = (G.REF / "train.py").read_text().splitlines()
    start = next(i for i, l in enumerate(lines) if l.strip().startswith("def make_cfg_model_fn("))
    indent = len(lines[start]) - len(lines[start].lstrip())
    end = start + 1
    while end < len(lines) and (not lines[end].strip() or len(lines[end]) - len(lines[end].lstrip()) > indent):
        end += 1
    ns = {"torch": torch, "cfg_scale": cfg_scale, "num_classes": num_classes}
    exec(textwrap.dedent("\n".join(lines[start:end])), ns)
    return ns["make_cfg_model_fn"]


def main():
    G._stub_missing()
    sys.path.insert(0, str(G.REF))
    import k_diffusion as K
    synth = G._load_synth()
    torch.set_num_threads(8)
    cfg = K.config.load_config(json.loads((G.REF / "configs" / "config_mnist_transformer.json").read_text()))
    inner = K.config.make_model(cfg).eval().requires_grad_(False)
    base = inner.state_dict()
    inner.load_state_dict(synth.synth_state_dict({k: v.shape for k, v in base.items()}, seed=1, base=base))
    model = K.config.make_denoiser_wrapper(cfg)(inner)
    num_classes = cfg["dataset"]["num_classes"]
    assert num_classes == 10
    g = torch.Generator().manual_seed(123)
    x = torch.randn(4, 1, 28, 28, generator=g) * 80                # the latent of tests/golden/cfg1_mnist.npz
    sigmas = K.sampling.get_sigmas_karras(10, 1e-2, 80)
    cc = torch.tensor([0, 3, 7, 9])
    sig = torch.tensor([0.3, 1.0, 5.0, 40.0])
    fn = reference_closure(3.0, num_classes)(model)
    assert reference_closure(1.0, num_classes)(model) is model
    with torch.no_grad():
        once = fn(x, sig, class_cond=cc)
        traj = K.sampling.sample_dpmpp_2m_sde(fn, x, sigmas, extra_args=dict(class_cond=cc), eta=0.0, solver_type="heun", disable=True,
                                              noise_sampler=lambda a, b: torch.zeros_like(x))
    np.savez(G.OUT / "cfg1_cfg.npz", class_cond=cc.numpy(), sigma=sig.numpy(), cfg_scale=3.0, num_classes=num_classes,
             model_fn=once.numpy(), dpmpp_2m_sde_heun_eta0=traj.numpy())
    print("wrote", G.OUT / "cfg1_cfg.npz", float(once.abs().mean()), float(traj.abs().mean()))


if __name__ == "__main__":
    main()
