#!/usr/bin/env python
"""(GPU) The EMA update of train.py's step: K.utils.ema_update (one kdb_ema_update launch) against the reference's per-tensor loop (one
lerp_ per parameter, one copy_ per buffer) on the parameter sets of cfg1 (MNIST transformer), the CIFAR-10 transformer and cfg2.

    python tools/ema_bench.py [--rounds 20] [--json out.json]

Each round times native, then the per-tensor loop, each call between CUDA events on the current stream after a device synchronise, so
the two routes alternate in one process; median and min-max over the rounds after two warm-up calls of each.  Achieved bytes/s counts
what the update must move: 12 bytes per parameter element (read the model's value and the average, write the average) and 8 per buffer
element (read, write), over the median time; the share of the H100 SXM data sheet's 3.35 TB/s HBM3 bandwidth is reported beside it.
The native call's time includes its host work (the table of every tensor pair, the version bumps); the device time of its
table copy and kernel (kdb_profile_* behind a gate that holds the stream until the call is enqueued, median over the rounds) and its bytes/s are reported beside it.  Both routes give the same bits (checked once per model).  The card's name, power limit and SM clock are read in the same call.
"""
import argparse
import copy
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "k-diffusion_b200")]
import torch

import k_diffusion as K

HBM_BYTES_PER_S = 3.35e12
CONFIGS = {"cfg1_mnist": ROOT / "tests/golden/cfg1_mnist_shapes.json", "cifar10_transformer": None,
           "cfg2_sw256": ROOT / "tests/golden/cfg2_sw256_shapes.json"}
# configs/config_cifar10_transformer.json of the reference
CIFAR10_TRANSFORMER = {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [32, 32], "patch_size": [2, 2],
                                 "depths": [2, 4], "widths": [256, 512], "self_attns": [{"type": "global"}, {"type": "global"}],
                                 "loss_config": "karras", "loss_weighting": "soft-min-snr", "dropout_rate": 0.05, "augment_prob": 0.12,
                                 "sigma_data": 0.5, "sigma_min": 0.01, "sigma_max": 80, "sigma_sample_density": {"type": "cosine-interpolated"}},
                       "dataset": {"type": "cifar10", "num_classes": 10}}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                         capture_output=True, text=True, check=True).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def build(name):
    path = CONFIGS[name]
    cfg = K.config.load_config(CIFAR10_TRANSFORMER if path is None else json.loads(path.read_text())["config"])
    torch.manual_seed(0)
    model = K.config.make_model(cfg).cuda()
    ema = copy.deepcopy(model)
    with torch.no_grad():
        for p in model.parameters():
            p.add_(torch.randn_like(p) * 1e-3)
    return model, ema


@torch.no_grad()
def per_tensor(model, ema, decay):
    """the reference's ema_update (utils.py:88-104)"""
    pe, be = dict(ema.named_parameters()), dict(ema.named_buffers())
    for k, p in model.named_parameters():
        pe[k].lerp_(p, 1 - decay)
    for k, b in model.named_buffers():
        be[k].copy_(b)


def timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ema_bench needs a CUDA device")
    decay = 0.999
    res = {"card": card(), "rounds": args.rounds, "decay": decay, "models": {}}
    for name in CONFIGS:
        model, ema = build(name)
        check = copy.deepcopy(ema)
        K.utils.ema_update(model, ema, decay)
        per_tensor(model, check, decay)
        same = all(torch.equal(a, b) for a, b in zip(ema.state_dict().values(), check.state_dict().values()))
        params = sum(p.numel() for p in model.parameters())
        buffers = sum(b.numel() for b in model.buffers())
        nbytes = 12 * params + 8 * buffers
        routes = {"native": lambda: K.utils.ema_update(model, ema, decay), "per_tensor": lambda: per_tensor(model, ema, decay)}
        for fn in routes.values():
            fn()
            fn()
        times = {k: [] for k in routes}
        kernel = []
        for _ in range(args.rounds):
            for k, fn in routes.items():
                times[k].append(timed(fn))
            with K._native.profile(gate_ms=5.0) as p:   # the stream parked until the call is enqueued: no host time in the interval
                routes["native"]()
            kernel.append(p.by_family["ema"][1])
        row = {"parameters": params, "buffers": buffers, "tensors": len(list(model.parameters())) + len(list(model.buffers())),
               "bytes": nbytes, "bit_identical": same}
        for k, ts in times.items():
            med = statistics.median(ts)
            row[k] = {"median_ms": med, "min_ms": min(ts), "max_ms": max(ts), "GB_per_s": nbytes / med / 1e6,
                      "share_of_3.35TB_per_s": nbytes / med / 1e-3 / HBM_BYTES_PER_S}
        kmed = statistics.median(kernel)
        row["kernel"] = {"median_ms": kmed, "min_ms": min(kernel), "max_ms": max(kernel), "GB_per_s": nbytes / kmed / 1e6,
                         "share_of_3.35TB_per_s": nbytes / kmed / 1e-3 / HBM_BYTES_PER_S}
        row["speedup"] = row["per_tensor"]["median_ms"] / row["native"]["median_ms"]
        res["models"][name] = row
        print(name, json.dumps(row), flush=True)
    res["card_after"] = card()
    print(json.dumps(res))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
