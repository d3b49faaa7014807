#!/usr/bin/env python
"""One training step of an image_transformer_v2 model: zero_grad, loss, backward and an AdamW step on param_groups.  The native path
(Denoiser.loss, then backward: one engine evaluation, the loss kernel and one kdb_model_forward_train; after the optimizer step the next
loss rebinds and re-finalizes the engine, as in training) at the fp32 and the tf32 training precision (set_train_precision), against the
oracle's torch eager autograd of the reference formula with the same optimizer, with TF32 off and with
torch.backends.cuda.matmul.allow_tf32 = True (what the reference's train.py:101 sets), all on the same GPU, with synth.py weights:

    cfg1     the MNIST class-conditional transformer, 28x28, B = 32, soft-min-snr
    cfg2     the oxford_flowers shifted-window transformer at 64x64, B = 8, soft-min-snr
    cifar10  the reference's config_cifar10_transformer (32x32, patch 2, widths 256 / 512, depths 2 / 4, global attention), B = 128
             (dropout off: the native path trains without dropout)
    mnist_unet    the reference's config_mnist image_v1 U-Net (28x28), B = 32, through KarrasAugmentWrapper (aug_cond zeros), dropout off
    cifar10_unet  the reference's config_cifar10 image_v1 U-Net (32x32), B = 128, the same
    cifar10_unet_variance  that U-Net with has_variance: true, B = 128: a DenoiserWithVariance step (kdb_unet_forward_variance,
             kdb_variance_loss, kdb_unet_forward_train_variance) against a Denoiser step on the same model, timed alternately

The U-Net cases have three legs: the native exact fp32 path (one kdb_unet_forward and one kdb_unet_forward_train per step) and the
oracle's torch eager autograd with TF32 off and with torch.backends.cuda.matmul.allow_tf32 and torch.backends.cudnn.allow_tf32 on; their
--profile splits a native step's GPU kernel time by kernel: unet_conv_kernel (the forward, the backward's recomputes and every input
gradient), wgrad_kernel + segsum_kernel (weight and bias gradients), the attention VJP, the AdaGN backward, and the rest.

    python tools/train_bench.py [--iters 10] [--rounds 3] [--warmup 3] [--cases cfg1,cifar10] [--profile]

The four legs are timed alternately, step by step (CUDA events around each step), in `rounds` rounds of `iters` steps each.  Prints one
JSON line per case: median, min and max milliseconds per step over all rounds, each round's medians, the time of one re-finalize after a
parameter change at each native precision, and the card's name and power limit.  --profile adds, from torch.profiler over a few native fp32
steps of its own, the share of the GPU kernel time spent in the token-stream GEMMs (forward, input and weight gradients)."""
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

CIFAR10 = {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [32, 32], "patch_size": [2, 2], "depths": [2, 4],
                     "widths": [256, 512], "self_attns": [{"type": "global"}, {"type": "global"}], "loss_config": "karras",
                     "loss_weighting": "soft-min-snr", "sigma_data": 0.5},
           "dataset": {"type": "cifar10", "num_classes": 10}}
CASES = {"cfg1": ("cfg1_mnist_shapes.json", None, 32), "cfg2": ("cfg2_sw256_shapes.json", [64, 64], 8), "cifar10": (None, None, 128)}
UNET_CASES = {"mnist_unet": ("mnist", 32), "cifar10_unet": ("cifar10", 128)}
UNET_KERNELS = {"conv (forward, recompute, input gradients)": ("unet_conv_kernel",), "weight and bias gradients": ("wgrad_kernel", "segsum_kernel"),
                "attention VJP": ("attn_vjp",), "AdaGN backward": ("unet_adagn_vjp_kernel",)}
GEMM_KERNELS = ("gemm_simt_kernel", "gemm_vjp_kernel", "wgrad_kernel", "wgrad_tf32_kernel", "unet_conv_tc_kernel")
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
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    for name in args.cases.split(","):
        if name == "cifar10_unet_variance":
            print(json.dumps(variance_case(args, gpu)), flush=True)
            continue
        if name in UNET_CASES:
            print(json.dumps(unet_case(name, args, gpu)), flush=True)
            continue
        fixture, size, B = CASES[name]
        cfg = json.loads((ROOT / "tests" / "golden" / fixture).read_text())["config"] if fixture else json.loads(json.dumps(CIFAR10))
        if size:
            cfg["model"]["input_size"] = size
        cfg = K.config.load_config(cfg)
        m = cfg["model"]
        inner = K.config.make_model(cfg)
        sd = synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, 3)
        inner.load_state_dict(sd)
        inner = inner.cuda().eval()
        model = K.config.make_denoiser_wrapper(cfg)(inner)
        inner_t = K.config.make_model(cfg)
        inner_t.load_state_dict(sd)
        inner_t = inner_t.cuda().eval().set_train_precision("tf32")
        model_t = K.config.make_denoiser_wrapper(cfg)(inner_t)
        g = torch.Generator().manual_seed(0)
        H, W = m["input_size"]
        x = (torch.randn(B, m["input_channels"], H, W, generator=g) * 0.5).cuda()
        noise = torch.randn(x.shape, generator=g).cuda()
        sigma = torch.exp(torch.randn(B, generator=g) * 1.2 - 0.4).cuda()
        kw = {"class_cond": torch.randint(0, cfg["dataset"]["num_classes"], (B,), generator=g).cuda()} if cfg["dataset"]["num_classes"] else {}

        def native_step(model, inner):
            opt = torch.optim.AdamW(inner.param_groups(1e-5), betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-3)

            def step():
                opt.zero_grad(set_to_none=True)
                model.loss(x, noise, sigma, **kw).mean().backward()
                opt.step()
            return step

        def refinalize_ms(inner):
            """one re-finalize of the engine after a parameter change (what every training step pays once)"""
            def go():
                with torch.no_grad():
                    next(inner.parameters()).add_(0.0)
                inner.engine()
            go()
            return stats([step_ms(go) for _ in range(5)])["median"]

        native, native_t = native_step(model, inner), native_step(model_t, inner_t)

        params = {k: v.cuda().requires_grad_(not k.endswith(BUFFERS)) for k, v in sd.items()}
        names = {id(p): k for k, p in inner.named_parameters()}
        topt = torch.optim.AdamW([dict(g, params=[params[names[id(p)]] for p in g["params"]]) for g in inner.param_groups(1e-5)],
                                 betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-3)
        sdat = m["sigma_data"]

        def oracle(tf32):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            topt.zero_grad(set_to_none=True)
            c_skip, c_out, c_in = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sigma, sdat)]
            noised = x + noise * sigma.view(-1, 1, 1, 1)
            with torch.device("cuda"):
                f = O.model_forward(params, m, noised * c_in, sigma, **kw)
            w = (sigma * sdat) ** 2 / (sigma ** 2 + sdat ** 2) ** 2
            (((f - (x - c_skip * noised) / c_out) ** 2).flatten(1).mean(1) * w).mean().backward()
            topt.step()
            torch.backends.cuda.matmul.allow_tf32 = False

        legs = {"native_fp32": native, "native_tf32": native_t, "torch_eager_fp32": lambda: oracle(False),
                "torch_eager_tf32": lambda: oracle(True)}
        for _ in range(args.warmup):
            for leg in legs.values():
                leg()
        ms = {k: [] for k in legs}
        for _ in range(args.rounds):
            for k in legs:
                ms[k].append([])
            for _ in range(args.iters):
                for k, leg in legs.items():
                    ms[k][-1].append(step_ms(leg))
        rec = dict(case=name, batch=B, size=[H, W], **{f"{k}_ms": stats(sum(v, [])) for k, v in ms.items()},
                   round_medians={k: [stats(r)["median"] for r in v] for k, v in ms.items()},
                   refinalize_ms=dict(fp32=refinalize_ms(inner), tf32=refinalize_ms(inner_t)), gpu=gpu)
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    native()
                torch.cuda.synchronize()
            total = gemm = 0.0
            for e in prof.key_averages():
                t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
                total += t
                gemm += t if any(g in e.key for g in GEMM_KERNELS) else 0.0
            rec["native_fp32_gemm_share"] = gemm / total if total else None
        print(json.dumps(rec), flush=True)


def timed_legs(legs, args):
    for _ in range(args.warmup):
        for leg in legs.values():
            leg()
    ms = {k: [] for k in legs}
    for _ in range(args.rounds):
        for k in legs:
            ms[k].append([])
        for _ in range(args.iters):
            for k, leg in legs.items():
                ms[k][-1].append(step_ms(leg))
    return ms


def unet_case(name, args, gpu):
    from oracle import unet_oracle as U
    ref, B = UNET_CASES[name]
    cfg = json.loads((ROOT / "tests" / "golden" / "unet_configs.json").read_text())[ref]["config"]
    cfg["model"]["dropout_rate"] = 0.0
    cfg = K.config.load_config(cfg)
    m = cfg["model"]
    model = K.config.make_model(cfg)
    inner = model.inner_model
    sd = synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, 3)
    inner.load_state_dict(sd)
    model = model.cuda().eval()
    den = K.config.make_denoiser_wrapper(cfg)(model)
    g = torch.Generator().manual_seed(0)
    H, W = m["input_size"]
    x = (torch.randn(B, m["input_channels"], H, W, generator=g) * 0.5).cuda()
    noise = torch.randn(x.shape, generator=g).cuda()
    sigma = torch.exp(torch.randn(B, generator=g) * 1.2 - 0.4).cuda()
    opt = torch.optim.AdamW(inner.param_groups(1e-5), betas=(0.95, 0.999), eps=1e-6, weight_decay=1e-3)

    def native():
        opt.zero_grad(set_to_none=True)
        den.loss(x, noise, sigma).mean().backward()
        opt.step()

    params = {k: v.cuda().requires_grad_(not k.endswith(("timestep_embed.weight", ".kernel"))) for k, v in sd.items()}
    names = {id(p): k for k, p in inner.named_parameters()}
    topt = torch.optim.AdamW([dict(g, params=[params[names[id(p)]] for p in g["params"]]) for g in inner.param_groups(1e-5)],
                             betas=(0.95, 0.999), eps=1e-6, weight_decay=1e-3)
    sdat = m["sigma_data"]

    def oracle(tf32):
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
        topt.zero_grad(set_to_none=True)
        c_skip, c_out, c_in = [c.view(-1, 1, 1, 1) for c in O.karras_scalings(sigma, sdat)]
        noised = x + noise * sigma.view(-1, 1, 1, 1)
        f = U.augment_forward(params, m, noised * c_in, sigma)
        w = (sigma * sdat) ** 2 / (sigma ** 2 + sdat ** 2) ** 2
        (((f - (x - c_skip * noised) / c_out) ** 2).flatten(1).mean(1) * w).mean().backward()
        topt.step()
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False

    legs = {"native_fp32": native, "torch_eager_fp32": lambda: oracle(False), "torch_eager_tf32": lambda: oracle(True)}
    ms = timed_legs(legs, args)

    def refinalize():
        with torch.no_grad():
            next(inner.parameters()).add_(0.0)
        inner.engine(True)
    refinalize()
    rec = dict(case=name, batch=B, size=[H, W], **{f"{k}_ms": stats(sum(v, [])) for k, v in ms.items()},
               round_medians={k: [stats(r)["median"] for r in v] for k, v in ms.items()},
               refinalize_ms=dict(fp32=stats([step_ms(refinalize) for _ in range(5)])["median"]), gpu=gpu)
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                native()
            torch.cuda.synchronize()
        share = {k: 0.0 for k in UNET_KERNELS}
        total = 0.0
        for e in prof.key_averages():
            t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            total += t
            for k, pats in UNET_KERNELS.items():
                if any(p in e.key for p in pats):
                    share[k] += t
                    break
        rec["native_fp32_kernel_share"] = {k: v / total for k, v in share.items()} if total else None
    return rec


def variance_case(args, gpu):
    """The learned-variance loss's cost: the same has_variance U-Net and AdamW step behind DenoiserWithVariance and behind Denoiser"""
    cfg = json.loads((ROOT / "tests" / "golden" / "unet_configs.json").read_text())["cifar10"]["config"]
    cfg["model"].update(dropout_rate=0.0, has_variance=True)
    cfg = K.config.load_config(cfg)
    m, B = cfg["model"], 128
    model = K.config.make_model(cfg)
    inner = model.inner_model
    inner.load_state_dict(synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, 3))
    model = model.cuda().eval()
    g = torch.Generator().manual_seed(0)
    H, W = m["input_size"]
    x = (torch.randn(B, m["input_channels"], H, W, generator=g) * 0.5).cuda()
    noise = torch.randn(x.shape, generator=g).cuda()
    sigma = torch.exp(torch.randn(B, generator=g) * 1.2 - 0.4).cuda()
    opt = torch.optim.AdamW(inner.param_groups(1e-5), betas=(0.95, 0.999), eps=1e-6, weight_decay=1e-3)

    def leg(den):
        def step():
            opt.zero_grad(set_to_none=True)
            den.loss(x, noise, sigma).mean().backward()
            opt.step()
        return step

    variance = K.config.make_denoiser_wrapper(cfg)(model)
    assert type(variance) is K.layers.DenoiserWithVariance
    legs = {"variance": leg(variance), "denoiser": leg(K.layers.Denoiser(model, m["sigma_data"], weighting=m["loss_weighting"]))}
    ms = timed_legs(legs, args)
    return dict(case="cifar10_unet_variance", batch=B, size=[H, W], **{f"{k}_ms": stats(sum(v, [])) for k, v in ms.items()},
                round_medians={k: [stats(r)["median"] for r in v] for k, v in ms.items()}, gpu=gpu)


if __name__ == "__main__":
    main()
