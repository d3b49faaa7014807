#!/usr/bin/env python
"""The reference's learned-variance training loss of the image_v1 U-Net as data, recorded from the REAL reference (build container only; the
absent third-party modules stubbed as make_golden.py does):

    K_DIFFUSION_REFERENCE=<checkout> python oracle/make_golden_unet_variance.py   # -> tests/golden/unet_variance.npz, unet_variance_meta.json

Cases: the has_variance edge config of tests/golden/unet_edges.json (KarrasAugmentWrapper), and a patch_size 2 + mapping_cond variant of it
without the wrapper, with synth.py weights (seed 3; proj_out nonzero, its variance row included) in eval mode and dropout_rate 0.  For each:
the inner model's logvar (return_variance=True) on the loss's noised input and the per-sample losses of the reference's
DenoiserWithVariance.loss, in float64 and fp32, and for every parameter the norm of its float64 gradient, its dot product with a fixed probe
and the relative L2 distance of the fp32 gradient from the float64 one (the reference's own fp32 error)."""
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np
import torch

import make_golden as G
from make_golden_unet_train import inputs, probe

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"


def cases():
    variance = json.loads((GOLDEN / "unet_edges.json").read_text())["variance"]["config"]
    patch2 = json.loads(json.dumps(variance))
    patch2["model"].update(patch_size=2, mapping_cond_dim=3, augment_wrapper=False, input_size=[16, 16])
    return {"variance": (variance, 2), "patch2_mcond": (patch2, 3)}


def main():
    G._stub_missing()
    sys.path.insert(0, str(G.REF))
    import k_diffusion as K
    synth = G._load_synth()
    torch.set_num_threads(8)
    rec, meta = {}, {"cases": {}, "configs": {}}
    for name, (cfg, B) in cases().items():
        c = K.config.load_config(json.loads(json.dumps(cfg)))
        c["model"]["dropout_rate"] = 0.0
        model = K.config.make_model(c)
        inner = model.inner_model if isinstance(model, K.augmentation.KarrasAugmentWrapper) else model
        inner.load_state_dict(synth.synth_state_dict({k: list(v.shape) for k, v in inner.state_dict().items()}, 3, {}))
        meta["configs"][name] = c
        x, noise, sigma, kw = inputs(c["model"], B, seed=21)
        grads = {}
        for dt in (torch.float64, torch.float32):
            model = model.to(dt).eval()
            den = K.config.make_denoiser_wrapper(c)(model)
            assert isinstance(den, K.layers.DenoiserWithVariance)
            xd, nd, sd_, kwd = x.to(dt), noise.to(dt), sigma.to(dt), {k: v.to(dt) for k, v in kw.items()}
            with torch.no_grad():
                c_in = den.get_scalings(sd_)[2].view(-1, 1, 1, 1)
                _, logvar = model((xd + nd * sd_.view(-1, 1, 1, 1)) * c_in, sd_, return_variance=True, **kwd)
            inner.zero_grad(set_to_none=True)
            loss = den.loss(xd, nd, sd_, **kwd)
            loss.sum().backward()
            rec[f"{name}_loss_{str(dt)[6:]}"] = loss.detach().double().numpy()
            rec[f"{name}_logvar_{str(dt)[6:]}"] = logvar.double().numpy()
            grads[dt] = {k: None if p.grad is None else p.grad.detach().double() for k, p in inner.named_parameters()}
        case = {}
        for k, g64 in grads[torch.float64].items():
            assert g64 is not None, k
            n = g64.norm().item()
            case[k] = dict(norm=n, probe=(g64 * probe(g64.shape, k)).sum().item(),
                           fp32_rel=(grads[torch.float32][k] - g64).norm().item() / n if n > 0 else 0.0)
        meta["cases"][name] = case
        for k, v in dict(x=x, noise=noise, sigma=sigma, **kw).items():
            rec[f"{name}_{k}"] = v.numpy()
    np.savez_compressed(GOLDEN / "unet_variance.npz", **rec)
    (GOLDEN / "unet_variance_meta.json").write_text(json.dumps(meta, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
