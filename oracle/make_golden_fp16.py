#!/usr/bin/env python
"""fp16 error budget of the image_v1 U-Net, measured on the REAL reference (checkout named by $K_DIFFUSION_REFERENCE):

    python oracle/make_golden_fp16.py        # -> tests/golden/fp16_budget.json

The recipe of oracle/make_golden_tf32.py with fp16 in place of tf32.  It runs the reference U-Net on the CPU twice on the inputs of
oracle/make_golden_unet.py (same synth weights, seeds, sigmas and call variants):

- plain fp32;
- with the arithmetic of the engine's fp16 precision: every Conv2d's input and weight rounded to the nearest fp16 (ties to even, +-inf
  past 65504) by forward pre-hooks, and the self-attention's q, k, v and softmax probabilities P rounded to fp16 -- the reference
  module's `F.scaled_dot_product_attention` is replaced at run time, in that module's namespace only, by a restatement that rounds them
  (scores and softmax in fp32).

It records rel_l2 = |fp16 - fp32|_2 / |fp32|_2 of the whole denoiser output for the four reference configs and the six edge configs at
every recorded call variant (B = 3 at sigma_min, 1, sigma_max), and of the mnist Heun-10 trajectory.  The GPU tests hold the engine's
fp16 route to twice these numbers (tests/test_gpu_unet_fp16.py); tests/test_unet_fp16_host.py checks that the oracle with the same
emulation reproduces them.
"""
import json
import math
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
import torch

from make_golden import OUT, REF, _load_synth, _stub_missing
from make_golden_tf32 import rel_l2
from make_golden_unet import CONFIGS, EDGE_BASE, EDGES, record


def f16_round(t):
    """t rounded to the nearest fp16 value (ties to even, +-inf past 65504) by way of fp32, as the engine rounds its fp32 operands"""
    return t.float().half().to(t.dtype)


def f16_sdpa(q, k, v, attn_mask=None, dropout_p=0.0, **kwargs):
    """scaled_dot_product_attention with q, k, v and the unnormalised probabilities P = exp(s - max s) rounded to fp16, divided by the
    sum of the rounded P (global attention, no mask, no dropout: what SelfAttention2d calls with the recorded dropout p = 0)"""
    assert attn_mask is None and dropout_p == 0.0 and not kwargs
    s = f16_round(q) @ f16_round(k).transpose(-2, -1) / math.sqrt(q.shape[-1])
    p = f16_round(torch.exp(s - s.amax(-1, keepdim=True)))
    return (p @ f16_round(v)) / p.sum(-1, keepdim=True)


class F16Namespace:
    """torch.nn.functional with scaled_dot_product_attention replaced by f16_sdpa"""

    def __init__(self, F):
        self._F = F

    def __getattr__(self, name):
        return f16_sdpa if name == "scaled_dot_product_attention" else getattr(self._F, name)


def fp16_mode(K, den):
    """context: den's Conv2d weights and inputs rounded to fp16, the reference's attention at fp16; restores everything on exit"""
    class Ctx:
        def __enter__(self):
            self.saved, self.hooks = [], []
            for mod in den.modules():
                if isinstance(mod, torch.nn.Conv2d):
                    self.saved.append((mod, mod.weight.data))
                    mod.weight.data = f16_round(mod.weight.data)
                    self.hooks.append(mod.register_forward_pre_hook(lambda m, args: (f16_round(args[0]),) + tuple(args[1:])))
            self.F = K.layers.F
            K.layers.F = F16Namespace(self.F)

        def __exit__(self, *exc):
            K.layers.F = self.F
            for h in self.hooks:
                h.remove()
            for mod, w in self.saved:
                mod.weight.data = w
    return Ctx()


def main():
    _stub_missing()
    sys.path.insert(0, str(REF))
    import k_diffusion as K
    synth = _load_synth()
    torch.set_num_threads(8)
    out = {"how": "reference image_v1 fp32 vs the same module with every Conv2d's input and weight rounded (nearest, ties to even) to fp16 "
                  "and the attention's q, k, v, P rounded to fp16; inputs, weights and seeds of oracle/make_golden_unet.py; "
                  "rel_l2 = |fp16 - fp32|_2 / |fp32|_2 over the whole output"}
    runs = [(name, K.config.load_config(json.loads((REF / "configs" / path).read_text())), 200 + seed)
            for seed, (name, path) in enumerate(CONFIGS.items())]
    for seed, (name, over) in enumerate(EDGES.items()):
        cfg = json.loads((REF / "configs" / EDGE_BASE).read_text())
        cfg["model"].update(over)
        runs.append(("edge_" + name, K.config.load_config(cfg), 300 + seed))
    for name, cfg, seed in runs:
        den, rec, _, g = record(K, synth, cfg, seed)
        keys = [k for k in rec if k.startswith("denoised")]
        with torch.no_grad(), fp16_mode(K, den):
            for key in keys:
                kw = {}
                if key in ("denoised_aug", "denoised_aug_mc"):
                    kw["aug_cond"] = rec["aug_cond"]
                if key.endswith("_mc"):
                    kw["mapping_cond"] = rec["mapping_cond"]
                out[f"{name}.{key}"] = rel_l2(den(rec["x"], rec["sigma"], **kw), rec[key])
        if name == "mnist":
            m = cfg["model"]
            c, (h, w) = m["input_channels"], m["input_size"]
            with torch.no_grad():
                xt = torch.randn(2, c, h, w, generator=g) * m["sigma_max"]
                sigmas = K.sampling.get_sigmas_karras(10, m["sigma_min"], m["sigma_max"])
                ref = K.sampling.sample_heun(den, xt, sigmas, disable=True)
                with fp16_mode(K, den):
                    low = K.sampling.sample_heun(den, xt, sigmas, disable=True)
            out["mnist.heun10"] = rel_l2(low, ref)
    (OUT / "fp16_budget.json").write_text(json.dumps(out, indent=1))
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
