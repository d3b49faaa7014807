#!/usr/bin/env python
"""Device time of the stand-alone tensor-core attention launches of the cfg2 model at its batch-32 shapes, against their hardware
bounds.  Run on the GPU box:

    python tools/attn_bench.py [--repeat 500] [--json out.json]

  window shift 0 / 4   the level-1 shifted-window launches: B = 32, 32 x 32 tokens, 4 heads of 64, 8 x 8 windows
  global               the middle-level global launches: B = 32, 16 x 16 tokens (256 keys per image), 8 heads of 64

Both run as the model runs them: bf16 qkv with cosine-normalised q and k, and the logit bound (the cosine-similarity scale) given, so
the softmax takes the fixed shift.  Each launch is timed on its own by CUDA events and a kernel's time is the median over --repeat
launches; the launches go straight to kdb_attention, so no torch op is inside the events.  Bounds: QK^T + PV FLOPs / 989 TFLOP/s and
minimum HBM bytes (qkv read once, output written once) / 3.35 TB/s (H100 SXM data sheet, dense BF16 and HBM3).  The library is the one
k_diffusion._native loads: $KDB200_LIB if set, so two builds can be compared by alternating calls.
"""
import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (str(ROOT), str(ROOT / "k-diffusion_b200"), str(ROOT / "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)
import torch

from fused_bench import row
from gemm_bench import gpu_info
from k_diffusion import _native as N_

B, SCALE = 32, 10.0
SHAPES = [  # name, h, w, heads, kind, shift
    ("window shift 0", 32, 32, 4, "shifted-window", 0),
    ("window shift 4", 32, 32, 4, "shifted-window", 4),
    ("global", 16, 16, 8, "global", 0),
]


def time_launches(launch, repeat):
    """median, min and max device time (us) of `launch()` over `repeat` launches"""
    for _ in range(10):
        launch()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(repeat)]
    for e0, e1 in ev:
        e0.record()
        launch()
        e1.record()
    torch.cuda.synchronize()
    ts = sorted(e0.elapsed_time(e1) * 1e3 for e0, e1 in ev)
    return ts[len(ts) // 2], ts[0], ts[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=500)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "attn_bench measures on the GPU"
    lib, st = N_.lib(), N_.stream()
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for name, h, w, nh, kind, shift in SHAPES:
        M, keys = B * h * w, (64 if kind == "shifted-window" else h * w)
        t = torch.randn(B, h * w, 3, nh, 64, device="cuda", generator=g)
        t[:, :, :2] = t[:, :, :2] / t[:, :, :2].norm(dim=-1, keepdim=True) * SCALE ** 0.5
        qkv = t.to(torch.bfloat16).reshape(B, h * w, 3 * nh * 64).contiguous()
        out = torch.empty(B, h * w, nh * 64, dtype=torch.bfloat16, device="cuda")
        bound = torch.full([nh], SCALE, device="cuda")
        code, param = N_._ATTN_CODE[kind], (8 if kind == "shifted-window" else 0)
        launch = lambda: N_.check(lib.kdb_attention(N_.PREC_BF16, 1, N_.ptr(qkv), N_.ptr(out), B, h, w, nh, 64, code, param, shift,
                                                    N_.ptr(bound), st))
        flop = 4.0 * M * keys * 64 * nh                                  # S = Q K^T and O = P V
        hbm = (qkv.numel() + out.numel()) * 2
        r = row(name, *time_launches(launch, a.repeat), flop, hbm)
        r["exp_m"] = round(M * keys * nh / 1e6, 1)
        rows.append(r)
    res = dict(gpu=gpu_info(), lib=str(N_.LIB_PATH), repeat=a.repeat, batch=B, kernels=rows)
    print(json.dumps(res["gpu"]), res["lib"])
    for r in rows:
        print(f"  {r['kernel']:16s} {r['us']:8.2f} us (min {r['us_min']:.2f}, max {r['us_max']:.2f})  {r['tflops']:6.1f} TFLOP/s  "
              f"MMA bound {r['mma_bound_us']:.2f} us  HBM bound {r['hbm_bound_us']:.2f} us ({r['hbm_mb']} MB)  {r['exp_m']} M exp")
    if a.json:
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
