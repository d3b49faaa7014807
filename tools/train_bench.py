#!/usr/bin/env python
"""One training step of an image_transformer_v2 model: zero_grad, loss, backward and an AdamW step on param_groups.  The native path
(Denoiser.loss, then backward: one fp32 engine evaluation, the loss kernel and one kdb_model_forward_train; after the optimizer step the
next loss rebinds and re-finalizes the engine, as in training) against the oracle's torch eager fp32 autograd of the reference formula with
the same optimizer, both on the same GPU, with synth.py weights:

    cfg1   the MNIST class-conditional transformer, 28x28, B = 32, soft-min-snr
    cfg2   the oxford_flowers shifted-window transformer at 64x64, B = 8, soft-min-snr

    python tools/train_bench.py [--iters 10] [--rounds 3] [--warmup 3]

The two are timed alternately, step by step (CUDA events around each step), in `rounds` rounds of `iters` pairs.  Prints one JSON line per
case: median, min and max milliseconds per step over all rounds, each round's medians, and the card's name and power limit."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (str(ROOT), str(ROOT / "k-diffusion_b200"), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch

import k_diffusion as K
from oracle import kdiff_oracle as O
from oracle.fixtures import synth_sd

CASES = {"cfg1": ("cfg1_mnist_shapes.json", None, 32), "cfg2": ("cfg2_sw256_shapes.json", [64, 64], 8)}
BUFFERS = ("pos_emb.freqs", "time_emb.weight", "aug_emb.weight")


def step_ms(step):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def stats(ms):
    ms = sorted(ms)
    return dict(median=ms[len(ms) // 2], min=ms[0], max=ms[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    for name, (fixture, size, B) in CASES.items():
        cfg = json.loads((ROOT / "tests" / "golden" / fixture).read_text())["config"]
        if size:
            cfg["model"]["input_size"] = size
        cfg = K.config.load_config(cfg)
        m = cfg["model"]
        inner = K.config.make_model(cfg)
        sd = synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, 3)
        inner.load_state_dict(sd)
        inner = inner.cuda().eval()
        model = K.config.make_denoiser_wrapper(cfg)(inner)
        g = torch.Generator().manual_seed(0)
        H, W = m["input_size"]
        x = (torch.randn(B, m["input_channels"], H, W, generator=g) * 0.5).cuda()
        noise = torch.randn(x.shape, generator=g).cuda()
        sigma = torch.exp(torch.randn(B, generator=g) * 1.2 - 0.4).cuda()
        kw = {"class_cond": torch.randint(0, cfg["dataset"]["num_classes"], (B,), generator=g).cuda()} if cfg["dataset"]["num_classes"] else {}

        opt = torch.optim.AdamW(inner.param_groups(1e-5), betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-3)

        def native():
            opt.zero_grad(set_to_none=True)
            model.loss(x, noise, sigma, **kw).mean().backward()
            opt.step()

        params = {k: v.cuda().requires_grad_(not k.endswith(BUFFERS)) for k, v in sd.items()}
        names = {id(p): k for k, p in inner.named_parameters()}
        topt = torch.optim.AdamW([dict(g, params=[params[names[id(p)]] for p in g["params"]]) for g in inner.param_groups(1e-5)],
                                 betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-3)
        sdat = m["sigma_data"]

        def oracle():
            topt.zero_grad(set_to_none=True)
            c_skip, c_out, c_in = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sigma, sdat)]
            noised = x + noise * sigma.view(-1, 1, 1, 1)
            with torch.device("cuda"):
                f = O.model_forward(params, m, noised * c_in, sigma, **kw)
            w = (sigma * sdat) ** 2 / (sigma ** 2 + sdat ** 2) ** 2
            (((f - (x - c_skip * noised) / c_out) ** 2).flatten(1).mean(1) * w).mean().backward()
            topt.step()

        for _ in range(args.warmup):
            native()
            oracle()
        nat, tor = [], []
        for _ in range(args.rounds):
            nat.append([])
            tor.append([])
            for _ in range(args.iters):
                nat[-1].append(step_ms(native))
                tor[-1].append(step_ms(oracle))
        rec = dict(case=name, batch=B, size=[H, W], native_ms=stats(sum(nat, [])), torch_eager_fp32_ms=stats(sum(tor, [])),
                   round_medians=dict(native=[stats(r)["median"] for r in nat], torch=[stats(r)["median"] for r in tor]), gpu=gpu)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
