#!/usr/bin/env python
"""(GPU) KID and FID on 50 000 seeded 2048-wide features: the native kernels against the reference's formulas in torch with TF32 off.

    python tools/metrics_bench.py [--n 50000] [--d 2048] [--rounds 5] [--json out.json]

Features are |N(0, 1)| draws (as post-ReLU Inception pool features are non-negative), x and y from one seed.  Each round times, in this
order, native kid, torch kid, native fid, torch fid -- each call ending in a device synchronise, CUDA events around it -- so the two
routes alternate in one process; medians with min and max over the rounds after one warm-up round.  The torch routes are the
reference's formulas (evaluation.py:93-161) restated on the same tensors, fp32 matmul with TF32 off.  Also reported: fid's d x d part
alone (two eigh square roots and the products, the same torch code in both routes), native kid's two kernels by device time
(kdb_profile_*), the FLOPs the native kid and the torch kid perform, computed from the shapes, and the results of both routes.  The
card's name, power limit and SM clock are read in the same call.
"""
import argparse
import json
import math
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "k-diffusion_b200")]
import torch

import k_diffusion as K


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                         capture_output=True, text=True, check=True).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def torch_kid(x, y, max_size=5000):
    def poly(a, b):
        return (a @ b.T / a.shape[-1] + 1) ** 3

    def mmd(a, b):
        m, n = a.shape[0], b.shape[0]
        kxx, kyy, kxy = poly(a, a), poly(b, b), poly(a, b)
        return ((kxx.sum() - kxx.diagonal().sum()) / m / (m - 1) + (kyy.sum() - kyy.diagonal().sum()) / n / (n - 1)
                - kxy.sum() * 2 / m / n)
    P = math.ceil(max(x.shape[0] / max_size, y.shape[0] / max_size))
    total = x.new_zeros([])
    for i in range(P):
        total = total + mmd(x[round(i * x.shape[0] / P):round((i + 1) * x.shape[0] / P)],
                            y[round(i * y.shape[0] / P):round((i + 1) * y.shape[0] / P)])
    return total / P


def cov_part(mx, cx, my, cy, eps=1e-8):
    eye = torch.eye(cx.shape[0], device=cx.device) * eps
    cx, cy = cx + eye, cy + eye
    sx = K.evaluation.sqrtm_eig(cx)
    return (mx - my).pow(2).sum() + torch.trace(cx + cy - 2 * K.evaluation.sqrtm_eig(sx @ cy @ sx))


def torch_fid(x, y):
    return cov_part(x.mean(0), torch.cov(x.T), y.mean(0), torch.cov(y.T))


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    v = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), float(v)


def kid_flops(sizes_x, sizes_y, d):
    """(native: upper triangles of k(x,x), k(y,y) and all of k(x,y) in 64-row tiles; torch: three full products), 2 FLOP per FMA"""
    nat = tor = 0
    for m, n in zip(sizes_x, sizes_y):
        tx, ty = -(-m // 64), -(-n // 64)
        nat += 2 * d * 64 * 64 * (tx * (tx + 1) // 2 + ty * (ty + 1) // 2 + tx * ty)
        tor += 2 * d * (m * m + n * n + m * n)
    return nat, tor


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000)
    ap.add_argument("--d", type=int, default=2048)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "metrics_bench needs a GPU"
    info = card()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(args.n, args.d, device="cuda", generator=g).abs_()
    y = torch.randn(args.n, args.d, device="cuda", generator=g).abs_() * 1.02
    E = K.evaluation
    routes = {"kid native": lambda: E.kid(x, y), "kid torch": lambda: torch_kid(x, y), "fid native": lambda: E.fid(x, y),
              "fid torch": lambda: torch_fid(x, y)}
    mx, cx = K._native.feature_mean_cov(x)
    my, cy = K._native.feature_mean_cov(y)
    routes["fid d x d part"] = lambda: cov_part(mx, cx, my, cy)
    times, values = {k: [] for k in routes}, {}
    for r in range(args.rounds + 1):
        for name, fn in routes.items():
            ms, v = timed(fn)
            values[name] = v
            if r > 0:
                times[name].append(ms)
    with K._native.profile() as p:
        E.kid(x, y)
        E.fid(x, y)
    torch.cuda.synchronize()
    P = math.ceil(args.n / 5000)
    bounds = E._partition_bounds(args.n, P)
    nat, tor = kid_flops(*[[b - a for a, b in zip(bounds, bounds[1:])]] * 2, args.d)
    out = {"card": info, "n": args.n, "d": args.d, "rounds": args.rounds,
           "ms": {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()},
           "values": values, "native_kernels_ms": {k: c_t[1] for k, c_t in p.by_family.items()},
           "kid_gflop": {"native": nat / 1e9, "torch": tor / 1e9},
           "kid_tflops": {"native": nat / statistics.median(times["kid native"]) / 1e9,
                          "torch": tor / statistics.median(times["kid torch"]) / 1e9},
           "card_after": card()}
    print(json.dumps(out, indent=1))
    if args.json:
        Path(args.json).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
