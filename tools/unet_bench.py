#!/usr/bin/env python
"""(GPU, fp32) Heun-50 on the image_v1 config_cifar10 U-Net: the native engine against torch eager fp32 of the same function.

    python tools/unet_bench.py [--batch 256] [--steps 50] [--json out.json]

Native: images/s of one graph-captured sample_heun call (warm-up call first, then the timed call ends in a device synchronise),
and the device time per kernel family of one eager denoiser evaluation (kdb_profile_*, stream gated so the launches run back to
back).  Torch: the oracle's functional model (oracle/unet_oracle.py) on the same card (cuDNN convolutions, TF32 disabled), the same
Heun loop (oracle/kdiff_oracle.py), timed the same way.  Synthetic seeded weights.  The card's name, power limit and SM clock are
read in the same call.
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
from oracle import kdiff_oracle as O
from oracle import unet_oracle as U
from oracle.fixtures import synth_sd


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    meta = json.loads((ROOT / "tests/golden/unet_configs.json").read_text())["cifar10"]
    cfg = K.config.load_config(meta["config"])
    sd = synth_sd(meta["shapes"], 1)
    model = K.config.make_model(cfg).eval().requires_grad_(False)
    model.load_state_dict(sd)
    den = K.config.make_denoiser_wrapper(cfg)(model.to("cuda"))
    m = cfg["model"]
    x = torch.randn(a.batch, 3, 32, 32, generator=torch.Generator().manual_seed(0)).cuda() * m["sigma_max"]
    sigmas = K.sampling.get_sigmas_karras(a.steps, m["sigma_min"], m["sigma_max"]).cuda()
    nfe = 2 * a.steps - 1
    res = {"card": card(), "workload": f"sample_heun {a.steps} steps ({nfe} evaluations), config_cifar10 image_v1, batch {a.batch}, fp32"}

    with torch.no_grad():
        K.sampling.sample_heun(den, x, sigmas, disable=True)                       # capture + warm-up
        native, t = timed(lambda: K.sampling.sample_heun(den, x, sigmas, disable=True))
        res["native"] = {"images_per_s": a.batch / t, "s_per_call": t, "ms_per_eval": 1e3 * t / nfe}
        sig = torch.full([a.batch], 2.0, device="cuda")
        den(x, sig)
        with K._native.profile(gate_ms=200.0) as p:
            den(x, sig)
        torch.cuda.synchronize()
        res["native"]["kernels_ms_per_eval"] = {f: {"launches": c, "ms": round(ms, 3)} for f, (c, ms) in
                                                sorted(p.by_family.items(), key=lambda kv: -kv[1][1])}

        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        sdc = {k: v.cuda() for k, v in U.strip_prefix(sd).items()}
        oden = U.make_denoiser(sdc, m)
        O.sample_heun(oden, x, sigmas[:3])                                          # warm-up of every shape
        eager, t = timed(lambda: O.sample_heun(oden, x, sigmas))
        res["torch_eager_fp32"] = {"images_per_s": a.batch / t, "s_per_call": t, "ms_per_eval": 1e3 * t / nfe,
                                   "settings": "cuDNN convolutions, TF32 off"}
        res["rel_l2_native_vs_eager"] = float((native - eager).double().norm() / eager.double().norm())
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if a.json:
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
