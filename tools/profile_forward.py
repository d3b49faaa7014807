#!/usr/bin/env python
"""Per-launch device times of ONE denoiser evaluation (eager launches, CUDA events after every kernel),
annotated with the GEMM shape each tensor-core launch corresponds to.  Run on the GPU box:

    python tools/profile_forward.py [--batch 32] [--precision bf16] [--json out.json] [--per-sample]

Default route = what the samplers (and bench.py) run: ONE shared conditioning row per evaluation, AdaRMSNorm folded into the
GEMMs (fold kernel + row statistics), launches enqueued behind a gate kernel so they execute back to back like a graph replay.
--per-sample profiles the route `model(x, sigma)` takes (per-sample conditioning rows, stand-alone RMSNorm kernels).
"""
import argparse
import json
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (str(ROOT), str(ROOT / "k-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch

import k_diffusion as K
from k_diffusion import _native


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--json", default=None)
    ap.add_argument("--config", default="sw", choices=["sw", "na", "c5"],
                    help="sw = cfg2 shifted-window model, na = cfg3/4 neighbourhood model, c5 = cfg5 (512x512, widths 256/512/1024; use --batch 16)")
    ap.add_argument("--per-sample", action="store_true")
    ap.add_argument("--repeat", type=int, default=1, help="evaluations inside the profiled region")
    args = ap.parse_args()
    fixture = "cfg2_sw256_shapes.json" if args.config == "sw" else "cfg3_na256_config.json"
    raw = json.loads((ROOT / "tests/golden" / fixture).read_text())["config"]
    if args.config == "c5":
        raw = {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [512, 512], "patch_size": [4, 4],
                         "depths": [2, 2, 4], "widths": [256, 512, 1024], "sigma_data": 0.5, "sigma_min": 1e-2, "sigma_max": 160}}
    cfg = K.config.load_config(raw)
    res = cfg["model"]["input_size"][0]
    inner = K.synth.synth_init_(K.config.make_model(cfg), seed=1).cuda().eval().set_precision(args.precision)
    model = K.Denoiser(inner, sigma_data=cfg["model"]["sigma_data"])
    x = torch.randn(args.batch, 3, res, res, device="cuda") * 10
    sig = torch.full([args.batch], 3.0, device="cuda")
    eng = inner.engine()
    table = eng.conditioning(sig[:1])

    def evaluate():
        if args.per_sample:
            return model(x, sig)
        return eng.forward(x, sig, table[0], 0, float(model.sigma_data), inner.resolved_precision())

    for _ in range(3):
        evaluate()
    torch.cuda.synchronize()
    with _native.profile(gate_ms=10.0 * args.repeat) as prof:
        for _ in range(args.repeat):
            evaluate()
    seq = K.models.flops.launch_layers(cfg["model"], args.batch, os.environ.get("KDB200_NO_FFN_FUSE", "0") != "1")
    gi = 0
    rows = []
    peak = 1396.9
    for fam, ms in prof.launches:
        note = ""
        if fam.startswith("gemm"):
            label, M, N, Kd, macs = seq[gi % len(seq)]
            tf = 2.0 * macs / (ms * 1e-3) / 1e12
            gi += 1
            gb = 2.0 * (M * Kd + N * Kd + M * (N if "geglu" not in label else N // 2) + (M * N if "res" in label else 0)) / (ms * 1e-3) / 1e9
            note = f"{label:18s} M={M:6d} N={N:5d} K={Kd:5d}  {tf:7.1f} TFLOP/s ({tf / peak:5.1%})  min-traffic {gb:7.0f} GB/s"
        rows.append((fam, ms, note))
        print(f"{fam:14s} {ms * 1000:9.1f} us  {note}")
    total = sum(ms for _, ms, _ in rows) / args.repeat
    print(f"route: {'per-sample conditioning' if args.per_sample else 'shared conditioning row, fused RMSNorm'}; {args.repeat} evaluation(s) profiled")
    print(f"total {total:.3f} ms per evaluation for batch {args.batch} -> {args.batch / total * 1000 / 99:.1f} img/s at 99 evaluations per image")
    by = {}
    for fam, ms, _ in rows:
        by[fam] = by.get(fam, 0) + ms / args.repeat
    for fam, ms in sorted(by.items(), key=lambda kv: -kv[1]):
        print(f"  {fam:14s} {ms:8.3f} ms  {ms / total:6.1%}")
    if args.json:
        Path(args.json).write_text(json.dumps(dict(batch=args.batch, precision=args.precision, total_ms=total,
                                                   launches=[dict(family=f, us=ms * 1000, note=n) for f, ms, n in rows]), indent=1))


if __name__ == "__main__":
    main()
