#!/usr/bin/env python
"""Cost of the reverse-mode derivative on the native engine: the fp32 forward, one kdb_model_forward_jvp and one kdb_model_forward_vjp,
and one guided Euler step (one forward under torch.autograd, one backward, one update), on cfg1 and the cfg2 model at 64x64 and 256x256,
all at B = 2.

    python tools/vjp_bench.py [--reps 7] [--json out.json]
Times are CUDA-event medians (with min / max) over --reps runs after warm-up; the GPU's name, power limit and SM clock are recorded with them.
"""
import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
from jvp_bench import gpu_info, median_ms, model_from  # noqa: E402

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "vjp_bench measures on the GPU"
    res = {"gpu": gpu_info(), "rows": []}
    g = torch.Generator().manual_seed(0)
    for stem, size in (("cfg1_mnist", None), ("cfg2_sw256", 64), ("cfg2_sw256", 256)):
        cfg, model = model_from(stem)
        C, (H, W) = cfg["model"]["input_channels"], cfg["model"]["input_size"]
        H, W = (size, size) if size else (H, W)
        x = (torch.randn(2, C, H, W, generator=g) * 0.5).cuda()
        v = torch.randn(x.shape, generator=g).cuda()
        proj = (torch.randn(16, x[0].numel(), generator=g) / x[0].numel() ** 0.5).cuda()
        sig = torch.tensor([0.7, 0.7], device="cuda")
        ea = dict(class_cond=torch.tensor([1, 9], device="cuda")) if model.inner_model.class_emb is not None else {}

        def guided_step():
            with torch.enable_grad():
                xg = x.detach().requires_grad_()
                den = model(xg, sig, **ea)
                loss = (den.flatten(1) @ proj.T).square().sum()
                grad = torch.autograd.grad(loss, xg)[0]
            d = (x - (den.detach() - grad * 0.49)) / 0.7
            return x + d * -0.1

        row = dict(model=stem, batch=2, size=[H, W])
        for label, fn in (("forward", lambda: model(x, sig, **ea)), ("forward_jvp", lambda: model.jvp(x, sig, v, **ea)),
                          ("forward_vjp", lambda: model.vjp(x, sig, v, **ea)), ("guided_euler_step", guided_step)):
            ms, lo, hi = median_ms(fn, a.reps)
            row[label + "_ms"], row[label + "_range_ms"] = ms, [lo, hi]
        res["rows"].append(row)
        labels = ("forward", "forward_jvp", "forward_vjp", "guided_euler_step")
        print(f"{stem} {H}x{W} B=2: " + ", ".join(f"{k} {row[k + '_ms']:.3f} ms [{row[k + '_range_ms'][0]:.3f}, {row[k + '_range_ms'][1]:.3f}]"
                                                 for k in labels), flush=True)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if a.json:
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    with torch.no_grad():
        main()
