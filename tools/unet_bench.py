#!/usr/bin/env python
"""(GPU) Heun-50 on the image_v1 config_cifar10 U-Net: the native engine against torch eager of the same function.

    python tools/unet_bench.py [--batch 256] [--steps 50] [--precision fp32|tf32|fp16] [--json out.json]

Native: images/s of one graph-captured sample_heun call (warm-up call first, then the timed call ends in a device synchronise),
and the device time per kernel family of one eager denoiser evaluation (kdb_profile_*, stream gated so the launches run back to
back).  --precision tf32 times the tf32 route and, in the same call, the fp32 route it is measured against.  Torch: the oracle's
functional model (oracle/unet_oracle.py) on the same card, the same Heun loop (oracle/kdiff_oracle.py), timed the same way, with
cuDNN / matmul TF32 off and, at --precision tf32, also on (torch's own default for cuDNN convolutions).  The convolution and
attention FLOPs of one evaluation are computed from the shapes; over the profiled time of their kernel families they are reported as a
share of the H100 SXM data-sheet dense TF32 rate (495 TFLOP/s) -- a share of a data-sheet figure, not a rate the card reached.
--precision fp16 times, in one call, the fp16, tf32 and fp32 native routes alternating (two rounds), then torch eager with TF32 on and
under autocast(float16); each leg reports images/s, the device time of one evaluation's convolutions, attention and AdaGN, and its
sample's rel-L2 against the native fp32 sample.  Synthetic seeded weights.  The card's name, power limit and SM clock are read in the same call.
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


TF32_DATASHEET_FLOPS = 495e12          # H100 SXM, dense TF32, at up to 700 W
FP16_DATASHEET_FLOPS = 989e12          # H100 SXM, dense FP16, at up to 700 W


def eval_flops(sd, m, B):
    """(convolution, attention) FLOPs of one evaluation: 2 M N K for every conv the engine runs on the tensor cores at tf32 (ResConvBlock
    3x3 convs and skip, qkv_proj, out_proj); 4 B T^2 C for each self-attention (q k^T and p v)"""
    H, W = m["input_size"]
    n = len(m["depths"])
    conv = attn = 0
    for k, w in sd.items():
        parts = k.split(".")
        if not (k.endswith(".weight") and w.ndim == 4 and parts[1] in ("d_blocks", "u_blocks") and ("main" in parts or parts[-2] in
                                                                                                  ("skip", "qkv_proj", "out_proj"))):
            continue
        level = int(parts[2]) if parts[1] == "d_blocks" else n - 1 - int(parts[2])
        h, wd = U.level_hw(m, H, W, level)
        conv += 2 * B * h * wd * w.shape[0] * w[0].numel()
        if parts[-2] == "qkv_proj":
            attn += 4 * B * (h * wd) ** 2 * w.shape[1]
    return conv, attn


def native_leg(den, model, precision, x, sigmas, B, nfe):
    model.set_precision(precision)
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


def kernel_split(fams):
    """ms per evaluation of the convolutions, the attention and AdaGN from kdb_profile's kernel families"""
    ms = lambda names: round(sum(v["ms"] for f, v in fams.items() if f in names), 3)
    return {"conv": ms({"unet_conv", "unet_conv_tf32", "unet_conv_fp16"}), "attention": ms({"attn_generic", "unet_attn_tf32", "unet_attn_fp16"}),
            "adagn": ms({"unet_adagn"})}


def torch_eager_leg(oden, x, sigmas, B, nfe, settings):
    """torch eager Heun of the oracle's functional model: images/s, and the device time of one evaluation's convolutions (aten::conv2d,
    which includes the depthwise resampling filters), attention (aten::scaled_dot_product_attention) and group norms (AdaGN) from
    torch.profiler in a separate run"""
    O.sample_heun(oden, x, sigmas[:3])                                              # warm-up of every shape
    out, t = timed(lambda: O.sample_heun(oden, x, sigmas))
    sig = torch.full([x.shape[0]], 2.0, device="cuda")
    oden(x, sig)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA, torch.profiler.ProfilerActivity.CPU]) as prof:
        oden(x, sig)
        torch.cuda.synchronize()
    ops = {e.key: e.device_time_total / 1e3 for e in prof.key_averages()}
    split = {"conv": ops.get("aten::conv2d", 0.0), "attention": ops.get("aten::scaled_dot_product_attention", 0.0),
             "adagn": ops.get("aten::group_norm", 0.0)}
    return out, {"images_per_s": B / t, "s_per_call": t, "ms_per_eval": 1e3 * t / nfe, "settings": settings,
                 "kernels_ms_per_eval": {k: round(v, 3) for k, v in split.items()}}


def fp16_comparison(den, model, sd, m, x, sigmas, B, nfe, conv_flops, attn_flops, rounds=2):
    """--precision fp16: the fp16, tf32 and fp32 native routes, alternating for `rounds` rounds (the samples and kernel times of the last
    round), then torch eager with TF32 on and under autocast(float16); every sample's rel-L2 against the native fp32 one"""
    legs, samples = {}, {}
    for _ in range(rounds):
        for prec in ("fp16", "tf32", "fp32"):
            samples[prec], r = native_leg(den, model, prec, x, sigmas, B, nfe)
            legs.setdefault(prec, []).append(r)
    ref = samples["fp32"]
    rel = lambda s: float((s - ref).double().norm() / ref.double().norm())
    res = {}
    for prec, rs in legs.items():
        r = dict(rs[-1])
        r["images_per_s_each_round"] = [q["images_per_s"] for q in rs]
        r["split_ms_per_eval"] = kernel_split(r["kernels_ms_per_eval"])
        r["rel_l2_vs_native_fp32"] = rel(samples[prec])
        res[f"native_{prec}"] = r
    for prec, peak in (("fp16", FP16_DATASHEET_FLOPS), ("tf32", TF32_DATASHEET_FLOPS)):
        sp = res[f"native_{prec}"]["split_ms_per_eval"]
        res[f"native_{prec}"]["share_of_datasheet"] = {
            "conv": conv_flops / (sp["conv"] * 1e-3) / peak, "attention": attn_flops / (sp["attention"] * 1e-3) / peak,
            "note": f"FLOPs from the shapes over the profiled kernel time, divided by the {peak / 1e12:.0f} TFLOP/s dense data-sheet "
                    "figure; not a reached rate"}
    res["speedup_fp16_vs_tf32_each_round"] = [t["s_per_call"] / f["s_per_call"] for f, t in zip(legs["fp16"], legs["tf32"])]
    sdc = {k: v.cuda() for k, v in U.strip_prefix(sd).items()}
    oden = U.make_denoiser(sdc, m)
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    out, res["torch_eager_tf32"] = torch_eager_leg(oden, x, sigmas, B, nfe, "cuDNN convolutions and matmuls, TF32 on")
    res["torch_eager_tf32"]["rel_l2_vs_native_fp32"] = rel(out)
    with torch.autocast("cuda", dtype=torch.float16):
        out, res["torch_eager_autocast_fp16"] = torch_eager_leg(oden, x, sigmas, B, nfe, "autocast(float16), TF32 on")
    res["torch_eager_autocast_fp16"]["rel_l2_vs_native_fp32"] = rel(out.float())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--precision", choices=["fp32", "tf32", "fp16"], default="fp32")
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
    res = {"card": card(), "workload": f"sample_heun {a.steps} steps ({nfe} evaluations), config_cifar10 image_v1, batch {a.batch}, "
                                       f"{a.precision}"}
    conv_flops, attn_flops = eval_flops(U.strip_prefix(sd), m, a.batch)
    res["flops_per_eval"] = {"conv": conv_flops, "attention": attn_flops}

    if a.precision == "fp16":
        with torch.no_grad():
            res.update(fp16_comparison(den, model, sd, m, x, sigmas, a.batch, nfe, conv_flops, attn_flops))
        res["card_after"] = card()
        print(json.dumps(res, indent=1))
        if a.json:
            Path(a.json).write_text(json.dumps(res, indent=1))
        return

    with torch.no_grad():
        native, res["native"] = native_leg(den, model, a.precision, x, sigmas, a.batch, nfe)
        fams = res["native"]["kernels_ms_per_eval"]
        # a share of the tf32 data-sheet rate only for the families that run on the tf32 tensor cores
        conv_ms = fams.get("unet_conv_tf32", {}).get("ms", 0.0)
        attn_ms = fams.get("unet_attn_tf32", {}).get("ms", 0.0)
        res["native"]["share_of_datasheet_tf32"] = {
            "conv": conv_flops / (conv_ms * 1e-3) / TF32_DATASHEET_FLOPS if conv_ms else None,
            "attention": attn_flops / (attn_ms * 1e-3) / TF32_DATASHEET_FLOPS if attn_ms else None,
            "note": "FLOPs from the shapes over the profiled time of the tf32 kernel families (unet_conv_tf32, unet_attn_tf32; None where "
                    "none ran), divided by the 495 TFLOP/s data-sheet figure; not a reached rate"}
        if a.precision == "tf32":
            native32, res["native_fp32"] = native_leg(den, model, "fp32", x, sigmas, a.batch, nfe)
            res["rel_l2_native_tf32_vs_fp32"] = float((native - native32).double().norm() / native32.double().norm())
            res["speedup_tf32_vs_native_fp32"] = res["native_fp32"]["s_per_call"] / res["native"]["s_per_call"]

        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        sdc = {k: v.cuda() for k, v in U.strip_prefix(sd).items()}
        oden = U.make_denoiser(sdc, m)
        O.sample_heun(oden, x, sigmas[:3])                                          # warm-up of every shape
        eager, t = timed(lambda: O.sample_heun(oden, x, sigmas))
        res["torch_eager_fp32"] = {"images_per_s": a.batch / t, "s_per_call": t, "ms_per_eval": 1e3 * t / nfe,
                                   "settings": "cuDNN convolutions, TF32 off"}
        res["rel_l2_native_vs_eager"] = float((native - eager).double().norm() / eager.double().norm())
        if a.precision == "tf32":
            torch.backends.cudnn.allow_tf32 = True
            torch.backends.cuda.matmul.allow_tf32 = True
            O.sample_heun(oden, x, sigmas[:3])
            eager_tf32, t = timed(lambda: O.sample_heun(oden, x, sigmas))
            res["torch_eager_tf32"] = {"images_per_s": a.batch / t, "s_per_call": t, "ms_per_eval": 1e3 * t / nfe,
                                       "settings": "cuDNN convolutions and matmuls, TF32 on"}
            res["speedup_tf32_vs_torch_eager_tf32"] = t / res["native"]["s_per_call"]
            res["rel_l2_native_tf32_vs_eager_fp32"] = res.pop("rel_l2_native_vs_eager")
            res["rel_l2_eager_tf32_vs_eager_fp32"] = float((eager_tf32 - eager).double().norm() / eager.double().norm())
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if a.json:
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
