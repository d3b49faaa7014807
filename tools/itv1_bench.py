#!/usr/bin/env python
"""(GPU) Heun-50 on image_transformer_v1 models: the native engine at bf16 and fp32 against torch eager of the same function.

    python tools/itv1_bench.py [--configs cifar 256] [--precisions bf16 fp32] [--batch-cifar 128] [--batch-256 8] [--steps 50] [--json out.json]

Two configs: `cifar`, the CIFAR-sized config of tests/golden/itv1_meta.json (32x32x3, patch 2, width 512, depth 8: 256 tokens), and
`256`, 256x256x3 with patch 4, width 512, depth 12 (4096 tokens).  Synthetic seeded weights (k_diffusion/synth.py).  For each, at bf16
and at fp32: images/s of one graph-captured sample_heun call (a warm-up call first, then the timed call ends in a device synchronise)
and the device time per kernel family of one eager denoiser evaluation (kdb_profile_*, the stream gated so that the launches run back
to back).  Torch: the oracle's functional model (oracle/itv1_oracle.py) on the same card under torch.autocast(bfloat16), the same
Heun loop (oracle/kdiff_oracle.py), timed the same way, and the relative L2 distance of each native result from it.  The card's name,
power limit and SM clocks are read in the same call, before and after.  The fp32 route's global attention is the exact SIMT kernel,
whose time grows with the square of the token count: at 4096 tokens a Heun-50 call takes minutes per image (--precisions bf16 skips it).
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "k-diffusion_b200")]
import torch

import k_diffusion as K
from oracle import itv1_oracle as V
from oracle import kdiff_oracle as O
from oracle.fixtures import synth_sd

CONFIG_256 = {"model": {"type": "image_transformer_v1", "input_channels": 3, "input_size": [256, 256], "patch_size": [4, 4], "width": 512,
                        "depth": 12, "sigma_data": 1.0, "sigma_min": 1e-2, "sigma_max": 160.0},
              "dataset": {"num_classes": 0}}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                         capture_output=True, text=True, check=True).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t


def config(name):
    if name == "cifar":
        return K.config.load_config(json.loads((ROOT / "tests/golden/itv1_meta.json").read_text())["configs"]["cifar"]["config"])
    return K.config.load_config(json.loads(json.dumps(CONFIG_256)))


def native_leg(den, model, precision, x, sigmas, B, nfe):
    model.set_precision(precision)
    K.sampling.clear_graph_cache()
    K.sampling.sample_heun(den, x, sigmas, disable=True)                           # capture + warm-up
    out, t = timed(lambda: K.sampling.sample_heun(den, x, sigmas, disable=True))
    res = {"images_per_s": B / t, "s_per_call": t, "ms_per_eval": 1e3 * t / nfe}
    sig = torch.full([B], 2.0, device="cuda")
    den(x, sig)
    with K._native.profile(gate_ms=200.0) as p:
        den(x, sig)
    torch.cuda.synchronize()
    res["kernels_ms_per_eval"] = {f: {"launches": c, "ms": round(ms, 3)} for f, (c, ms) in sorted(p.by_family.items(), key=lambda kv: -kv[1][1])}
    return out, res


def bench(name, B, steps, precisions):
    cfg = config(name)
    model = K.config.make_model(cfg).eval().requires_grad_(False)
    sd = synth_sd({k: list(v.shape) for k, v in model.state_dict().items()}, 1)
    model.load_state_dict(sd)
    den = K.config.make_denoiser_wrapper(cfg)(model.to("cuda"))
    m = cfg["model"]
    c, (h, w) = m["input_channels"], m["input_size"]
    x = torch.randn(B, c, h, w, generator=torch.Generator().manual_seed(0)).cuda() * m["sigma_max"]
    sigmas = K.sampling.get_sigmas_karras(steps, m["sigma_min"], m["sigma_max"]).cuda()
    nfe = 2 * steps - 1
    tokens = (h // m["patch_size"][0]) * (w // m["patch_size"][1])
    res = {"workload": f"sample_heun {steps} steps ({nfe} evaluations), {h}x{w}x{c}, patch {m['patch_size']}, width {m['width']}, "
                       f"depth {m['depth']}, {tokens} tokens, batch {B}"}
    with torch.no_grad():
        outs = {}
        for precision in precisions:
            outs[precision], res[f"native_{precision}"] = native_leg(den, model, precision, x, sigmas, B, nfe)
            print(f"{name} native {precision}: {res[f'native_{precision}']['images_per_s']:.2f} images/s", file=sys.stderr, flush=True)
        oden = V.make_denoiser({k: v.cuda() for k, v in sd.items()}, m)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            O.sample_heun(oden, x, sigmas[:3])                                      # warm-up of every shape
            eager, t = timed(lambda: O.sample_heun(oden, x, sigmas))
        res["torch_eager_bf16_autocast"] = {"images_per_s": B / t, "s_per_call": t, "ms_per_eval": 1e3 * t / nfe}
        print(f"{name} torch eager: {B / t:.2f} images/s", file=sys.stderr, flush=True)
        for precision in precisions:
            res[f"native_{precision}"]["speedup_vs_torch_eager"] = t / res[f"native_{precision}"]["s_per_call"]
            res[f"native_{precision}"]["rel_l2_vs_torch_eager"] = float((outs[precision] - eager.float()).double().norm() /
                                                                       eager.double().norm())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", choices=["cifar", "256"], default=["cifar", "256"])
    ap.add_argument("--precisions", nargs="+", choices=["bf16", "fp32"], default=["bf16", "fp32"])
    ap.add_argument("--batch-cifar", type=int, default=128)
    ap.add_argument("--batch-256", type=int, default=8)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "itv1_bench.py measures on a GPU"
    res = {"card": card()}
    for name in a.configs:
        res[name] = bench(name, a.batch_cifar if name == "cifar" else a.batch_256, a.steps, a.precisions)
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if a.json:
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
