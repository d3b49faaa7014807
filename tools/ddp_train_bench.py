#!/usr/bin/env python
"""Median step time of native training under torch DistributedDataParallel: zero_grad, Denoiser.loss on the DDP-wrapped model, backward
(one native engine call, then DDP's all-reduce of every gradient), an AdamW step on param_groups and ema_update into a DDP-wrapped EMA
model, as train.py runs it under Accelerate.  NCCL, one rank per GPU, at world size 1 and at every larger world size the visible GPUs
allow; at world size 1 the same step also runs without the DDP wrapper, which prices the wrapper itself.  The batch is per rank, so
perfect scaling keeps the step time constant:

    cfg1        the MNIST class-conditional transformer, 28x28, B = 32 per rank, synth.py weights
    mnist_unet  the reference's config_mnist image_v1 U-Net (28x28) through KarrasAugmentWrapper, B = 32 per rank, dropout off

    python tools/ddp_train_bench.py [--iters 30] [--warmup 5] [--cases cfg1,mnist_unet] [--batch 32]

Prints one JSON line per case and world size (rank 0's median, min and max milliseconds per step, CUDA events around each step, the
ranks synchronised by a barrier before each step), and the card's name and power limit.  With one visible GPU it says so and reports
no scaling figure."""
import argparse
import datetime
import json
import os
import socket
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (str(ROOT), str(ROOT / "k-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

GOLDEN = ROOT / "tests" / "golden"


def build(case, device):
    import k_diffusion as K
    from oracle.fixtures import synth_sd
    if case == "cfg1":
        cfg = json.loads((GOLDEN / "cfg1_mnist_shapes.json").read_text())["config"]
    else:
        cfg = json.loads((GOLDEN / "unet_configs.json").read_text())["mnist"]["config"]
        cfg["model"]["dropout_rate"] = 0.0
    cfg = K.config.load_config(cfg)
    outer = K.config.make_model(cfg)
    inner = outer.inner_model if isinstance(outer, K.augmentation.KarrasAugmentWrapper) else outer
    inner.load_state_dict(synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, 3))
    return cfg, outer.to(device).eval(), inner


def stats(ms):
    ms = sorted(ms)
    return dict(median=ms[len(ms) // 2], min=ms[0], max=ms[-1])


def measure(case, device, args, wrap):
    import k_diffusion as K
    from torch.nn.parallel import DistributedDataParallel as DDP
    cfg, outer, inner = build(case, device)
    _, ema_outer, _ = build(case, device)
    model, ema = (DDP(outer, device_ids=[device.index]), DDP(ema_outer, device_ids=[device.index])) if wrap else (outer, ema_outer)
    den = K.config.make_denoiser_wrapper(cfg)(model)
    opt = torch.optim.AdamW(inner.param_groups(1e-5), betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-3)
    m = cfg["model"]
    g = torch.Generator().manual_seed(dist.get_rank() if wrap else 0)
    B, (H, W) = args.batch, m["input_size"]
    x = (torch.randn(B, m["input_channels"], H, W, generator=g) * 0.5).to(device)
    noise = torch.randn(x.shape, generator=g).to(device)
    sigma = torch.exp(torch.randn(B, generator=g) * 1.2 - 0.4).to(device)
    kw = {"class_cond": torch.randint(0, 10, (B,), generator=g).to(device)} if cfg["dataset"]["num_classes"] else {}

    def step():
        opt.zero_grad(set_to_none=True)
        den.loss(x, noise, sigma, **kw).mean().backward()
        opt.step()
        K.utils.ema_update(model, ema, 0.999)

    ms = []
    for i in range(args.warmup + args.iters):
        dist.barrier()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        torch.cuda.synchronize()
        if i >= args.warmup:
            ms.append(a.elapsed_time(b))
    return stats(ms)


def worker(rank, world, port, args, gpu):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    device = torch.device("cuda", rank)
    torch.cuda.set_device(device)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device, timeout=datetime.timedelta(minutes=10))
    for case in args.cases.split(","):
        rec = dict(case=case, world_size=world, batch_per_rank=args.batch, ddp_ms=measure(case, device, args, True))
        if world == 1:
            rec["no_ddp_ms"] = measure(case, device, args, False)
        if rank == 0:
            print(json.dumps(dict(rec, gpu=gpu)), flush=True)
    dist.barrier()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--cases", default="cfg1,mnist_unet")
    args = ap.parse_args()
    n = torch.cuda.device_count()
    if n == 0:
        raise SystemExit("ddp_train_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    gpu = [line.strip() for line in gpu.splitlines()][:n]
    if n == 1:
        print(json.dumps(dict(note="one GPU visible: world size 1 only, no scaling figure")), flush=True)
    for world in range(1, n + 1):
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        mp.spawn(worker, args=(world, port, args, gpu), nprocs=world, join=True)


if __name__ == "__main__":
    main()
