#!/usr/bin/env python
"""Per-call overhead of the external model wrappers (k_diffusion.external) around a trivial inner model that returns a fixed tensor:
the native wrapper (kdb_external_scale_in + kdb_external_combine) against the reference's torch formula (oracle/external_oracle.py),
both on the GPU, at the sizes their users run:

    sd   CompVisDenoiser, Stable Diffusion latents B = 8, 4x64x64, the model returning fp16 eps
    gd   OpenAIDenoiser, guided-diffusion 256x256 at B = 8, the model returning 6 channels (eps + learned variance), fp32

    python tools/external_bench.py [--iters 500] [--warmup 50]

Prints one JSON line per case: microseconds per call (host clock around `iters` calls ending in a device synchronise), kdb launches
per call, whether the two outputs are bit-identical, and the card's name and power limit."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (str(ROOT), str(ROOT / "k-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch

import k_diffusion as K
from k_diffusion import _native
from oracle import external_oracle as E


class FixedOutput(torch.nn.Module):
    """An inner model that costs nothing: it returns the same precomputed tensor whatever it is given."""

    def __init__(self, out):
        super().__init__()
        self.out = out
        self.register_buffer("alphas_cumprod", E.sd_alphas_cumprod())

    def forward(self, x, t, cond=None):
        return self.out

    def apply_model(self, x, t, cond):
        return self.out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name()


def time_calls(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters * 1e6


def case(name, ours, oracle, x, sigma, kw, iters, warmup):
    with torch.no_grad():
        same = torch.equal(ours(x, sigma, **kw), oracle(x, sigma, **kw))
        n0 = _native.launch_count()
        ours(x, sigma, **kw)
        launches = _native.launch_count() - n0
        us = {}
        for rep in range(3):                                 # alternate the two, keep each one's best
            for label, fn in (("native", ours), ("torch", oracle)):
                t = time_calls(lambda: fn(x, sigma, **kw), iters, warmup)
                us[label] = min(us.get(label, t), t)
    return dict(case=name, shape=list(x.shape), native_us_per_call=round(us["native"], 2), torch_us_per_call=round(us["torch"], 2),
                speedup=round(us["torch"] / us["native"], 3), launches_per_call=launches, bit_identical=same, card=card())


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("external_bench needs a GPU")
    dev = "cuda"
    g = torch.Generator().manual_seed(0)
    B = 8
    # Stable Diffusion: fp16 eps, quantize off, per-sample sigmas in the table's range
    x = (torch.randn(B, 4, 64, 64, generator=g) * 14.6).to(dev)
    sigma = torch.linspace(14.6, 0.03, B).to(dev)
    cond = torch.randn(B, 77, 768, generator=g).to(dev)
    inner = FixedOutput(torch.randn(B, 4, 64, 64, generator=g).to(dev, torch.float16)).to(dev)
    rows = [case("sd CompVisDenoiser fp16 eps", K.external.CompVisDenoiser(inner).to(dev), E.CompVisDenoiserOracle(inner), x, sigma,
                 dict(cond=cond), a.iters, a.warmup)]
    # guided diffusion: 6 output channels, eps read in place from the first 3
    x = (torch.randn(B, 3, 256, 256, generator=g) * 80).to(dev)
    sigma = torch.linspace(80.0, 0.03, B).to(dev)
    inner = FixedOutput(torch.randn(B, 6, 256, 256, generator=g).to(dev)).to(dev)
    rows.append(case("gd OpenAIDenoiser learned sigmas", K.external.OpenAIDenoiser(inner, E.ToyDiffusion(), device=dev),
                     E.OpenAIDenoiserOracle(inner, E.ToyDiffusion(), device=dev), x, sigma, {}, a.iters, a.warmup))
    for r in rows:
        print(json.dumps(r))


if __name__ == "__main__":
    main()
