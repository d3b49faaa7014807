#!/usr/bin/env python
"""Cost of the Hutchinson divergence term of log_likelihood on the native engine: one right-hand side of the likelihood ODE by the
4th-order finite difference (five fp32 forwards) against the forward-mode derivative (one kdb_model_forward_jvp), and the end-to-end
log_likelihood on cfg1 with both.

    python tools/jvp_bench.py [--reps 7] [--json out.json]
Times are CUDA-event medians over --reps runs after warm-up; the GPU's name, power limit and SM clock are recorded with them.
"""
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
from oracle.fixtures import synth_sd

S = K.sampling


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return dict(zip(q.split(","), (s.strip() for s in out.splitlines()[0].split(","))))
    except (OSError, subprocess.CalledProcessError):
        return {"name": torch.cuda.get_device_name()}


def model_from(stem):
    meta = json.loads((ROOT / "tests" / "golden" / f"{stem}_shapes.json").read_text())
    cfg = K.config.load_config(meta["config"])
    inner = K.config.make_model(cfg)
    inner.load_state_dict(synth_sd(meta["shapes"], 1))
    return cfg, K.config.make_denoiser_wrapper(cfg)(inner.to("cuda").eval().set_precision("fp32"))


def median_ms(fn, reps, inner=5):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(inner):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / inner)
    return sorted(ts)[len(ts) // 2], min(ts), max(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "jvp_bench measures on the GPU"
    res = {"gpu": gpu_info(), "rhs": [], "log_likelihood": []}
    g = torch.Generator().manual_seed(0)
    for stem, size in (("cfg1_mnist", None), ("cfg2_sw256", 64), ("cfg2_sw256", 256)):
        cfg, model = model_from(stem)
        C, (H, W) = cfg["model"]["input_channels"], cfg["model"]["input_size"]
        H, W = (size, size) if size else (H, W)
        x = (torch.randn(2, C, H, W, generator=g) * 0.5).cuda()
        v = (torch.randint(0, 2, x.shape, generator=g).float() * 2 - 1).cuda()
        ea = dict(class_cond=torch.tensor([1, 9], device="cuda")) if model.inner_model.class_emb is not None else {}
        y = (x, torch.zeros(2, device="cuda"))
        row = dict(model=stem, batch=2, size=[H, W])
        for label, jvp in (("fd_5_forwards", False), ("jvp", True)):
            rhs, _ = S._likelihood_rhs(model, x, ea, v, 1e-2, jvp=jvp)
            ms, lo, hi = median_ms(lambda: rhs(0.7, y), a.reps)
            row[label + "_ms"], row[label + "_range_ms"] = ms, [lo, hi]
        row["fd_over_jvp"] = row["fd_5_forwards_ms"] / row["jvp_ms"]
        res["rhs"].append(row)
        print(f"{stem} {H}x{W} B=2: rhs FD {row['fd_5_forwards_ms']:.3f} ms, JVP {row['jvp_ms']:.3f} ms ({row['fd_over_jvp']:.2f}x)", flush=True)
    cfg, model = model_from("cfg1_mnist")
    x = (torch.randn(2, 1, 28, 28, generator=g) * 0.4 + 0.1).cuda()
    v = (torch.randint(0, 2, x.shape, generator=g).float() * 2 - 1).cuda()
    ea = dict(class_cond=torch.tensor([1, 9], device="cuda"))
    for label, jvp in (("fd_5_forwards", False), ("jvp", True)):
        S.log_likelihood(model, x, 1e-2, 80., extra_args=ea, v=v, jvp=jvp)           # warm-up
        ts, info = [], None
        for _ in range(max(3, a.reps // 2)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ll, info = S.log_likelihood(model, x, 1e-2, 80., extra_args=ea, v=v, jvp=jvp)
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        res["log_likelihood"].append(dict(model="cfg1_mnist", batch=2, method=label, ms=sorted(ts)[len(ts) // 2], range_ms=[min(ts), max(ts)],
                                          fevals=info["fevals"], ll=[float(t) for t in ll]))
        print(f"cfg1 log_likelihood ({label}): {sorted(ts)[len(ts) // 2]:.1f} ms, fevals {info['fevals']}, ll {ll.tolist()}", flush=True)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if a.json:
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
