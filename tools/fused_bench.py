#!/usr/bin/env python
"""Device time of the two fused level-0 kernels of the cfg2 model at its batch-32 shapes, against their hardware bounds.  Run on the GPU box:

    python tools/fused_bench.py [--repeat 200] [--json out.json]

  attn_block  gemm_wg_attn_block_kernel (tc_attn_block.cuh): B = 32, 64 x 64 tokens, C = 128, shift 0 and 4
  ffn_fused   ffn_fused_kernel (tc_ffn_fused.cuh): M = 32 * 64 * 64 = 131072, C = 128, d_ff = 384

Each launch is timed on its own by CUDA events (the x it updates in place is restored from a pristine copy between launches, outside
the events); a kernel's time is the median over --repeat launches.  The launches go straight to the library entry points with the
interleaved up projection and the RoPE table prepared once, so no torch op is inside the events.  Bounds: FLOPs / 989 TFLOP/s and
minimum HBM bytes / 3.35 TB/s (H100 SXM data sheet, dense BF16 and HBM3); for ffn_fused also the bytes of weights every 128-row tile
streams from L2.  The library is the one k_diffusion._native loads: $KDB200_LIB if set, so two builds can be compared by alternating calls.
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

from gemm_bench import PEAK_TBS, PEAK_TFLOPS, gpu_info
from k_diffusion import _native as N_
from oracle import kdiff_oracle as O

B, H, W, C, DFF = 32, 64, 64, 128, 384
M = B * H * W


def time_launches(launch, x, x0, repeat):
    """median device time (us) of `launch()` over `repeat` launches, x restored from x0 before each"""
    for _ in range(5):
        x.copy_(x0)
        launch()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(repeat)]
    for e0, e1 in ev:
        x.copy_(x0)
        e0.record()
        launch()
        e1.record()
    torch.cuda.synchronize()
    ts = sorted(e0.elapsed_time(e1) * 1e3 for e0, e1 in ev)
    return ts[len(ts) // 2], ts[0], ts[-1]


def row(name, us, lo, hi, flop, hbm_bytes, l2_bytes=None):
    t_mma, t_hbm = flop / (PEAK_TFLOPS * 1e12) * 1e6, hbm_bytes / (PEAK_TBS * 1e12) * 1e6
    r = dict(kernel=name, us=round(us, 2), us_min=round(lo, 2), us_max=round(hi, 2), gflop=round(flop / 1e9, 2), tflops=round(flop / us / 1e6, 1),
             hbm_mb=round(hbm_bytes / 1e6, 1), mma_bound_us=round(t_mma, 2), hbm_bound_us=round(t_hbm, 2))
    if l2_bytes is not None:
        r["l2_weight_mb"] = round(l2_bytes / 1e6, 1)
        r["l2_weight_gbs"] = round(l2_bytes / us / 1e3)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=200)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "fused_bench measures on the GPU"
    lib, st = N_.lib(), N_.stream()
    g = torch.Generator(device="cuda").manual_seed(0)
    x0 = (torch.randn(M, C, device="cuda", generator=g) * 2).to(torch.bfloat16)
    x = x0.clone()
    ss = torch.zeros(M, 8, device="cuda")
    ss[:, 0] = x0.float().pow(2).sum(1)
    ss_out = torch.zeros(M, 8, device="cuda")
    rows = []

    # ---- attention block
    w_qkv = (torch.randn(3 * C, C, device="cuda", generator=g) / C ** 0.5).to(torch.bfloat16)
    w_out = (torch.randn(C, C, device="cuda", generator=g) / C ** 0.5).to(torch.bfloat16)
    scale = torch.tensor([10.0, 6.5], device="cuda")
    th = O.rope_theta(O.make_axial_pos(H, W), O.rope_freqs(64, 2)).to("cuda").float().reshape(H * W, 2, 8, 2).permute(1, 2, 0, 3)
    table = torch.cat([th.cos(), th.sin()], dim=-1).contiguous()      # as _native.attn_block_bf16 prepares it
    nwin = B * (H // 8) * (W // 8)
    attn_flop = 2.0 * nwin * 64 * (3 * C * C + 2 * 2 * 64 * 64 + C * C)          # qkv, S and P V of two heads, out_proj
    attn_bytes = 2 * M * C * 2 + 2 * M * 4 + (3 * C * C + C * C) * 2             # x in + out, sum(x^2) slot in + out, weights
    for shift in (0, 4):
        launch = lambda: N_.check(lib.kdb_attn_block_bf16(N_.ptr(x), N_.ptr(w_qkv), N_.ptr(w_out), N_.ptr(table), N_.ptr(scale), B, H, W, shift,
                                                           N_.ptr(ss), N_.ptr(ss_out), st))
        rows.append(row(f"attn_block shift {shift}", *time_launches(launch, x, x0, a.repeat), attn_flop, attn_bytes))

    # ---- feed-forward block
    w_up = (torch.randn(2 * DFF, C, device="cuda", generator=g) / C ** 0.5).to(torch.bfloat16)
    w_il = N_.interleave_geglu_rows(w_up)
    w_dn = (torch.randn(C, DFF, device="cuda", generator=g) / DFF ** 0.5).to(torch.bfloat16)
    launch = lambda: N_.check(lib.kdb_ffn_fused_bf16(N_.ptr(x), N_.ptr(w_il), N_.ptr(w_dn), M, DFF, N_.ptr(ss), N_.ptr(ss_out), st))
    ffn_flop = 2.0 * M * C * 3 * DFF                                              # up (2 d_ff outputs) + down
    ffn_bytes = 2 * M * C * 2 + 2 * M * 4 + 3 * DFF * C * 2
    ffn_l2 = (M // 128) * 3 * DFF * C * 2                                         # Wup + Wdown per 128-row tile
    rows.append(row("ffn_fused", *time_launches(launch, x, x0, a.repeat), ffn_flop, ffn_bytes, ffn_l2))

    res = dict(gpu=gpu_info(), lib=str(N_.LIB_PATH), repeat=a.repeat, kernels=rows)
    print(json.dumps(res["gpu"]), res["lib"])
    for r in rows:
        extra = f"  L2 weight stream {r['l2_weight_mb']} MB = {r['l2_weight_gbs']} GB/s" if "l2_weight_mb" in r else ""
        print(f"  {r['kernel']:20s} {r['us']:8.2f} us (min {r['us_min']:.2f}, max {r['us_max']:.2f})  {r['tflops']:6.1f} TFLOP/s  "
              f"MMA bound {r['mma_bound_us']:.2f} us  HBM bound {r['hbm_bound_us']:.2f} us ({r['hbm_mb']} MB){extra}")
    if a.json:
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
